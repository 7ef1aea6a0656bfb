/* mmssl_b200 -- C ABI of the H100-native MMSSL hot path (libmmssl_b200.so, sm_90a only).
 *
 * Plain pointers and sizes; no torch types.  Every pointer is a DEVICE pointer unless it is a
 * small descriptor struct/array marked "host".  `stream` is a cudaStream_t passed as void*.
 * All functions are asynchronous on `stream`, never synchronise, are CUDA-graph capturable, and
 * return 0 on success / non-zero on failure (message: mmssl_last_error()).  Matrices are
 * row-major fp32 with an explicit leading dimension (in floats).
 *
 * Each entry point names the reference code it replaces (paths relative to
 * MMSSL/ of the reference repository).  The reference itself is Python on stock torch ops, so the
 * "reference-side binding" is the ctypes stub in mmssl_b200/_lib.py (see INTEGRATION.md).
 */
#ifndef MMSSL_B200_H
#define MMSSL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MMSSL_ABI_VERSION 1
#define MMSSL_SPMM_MAX_RHS 3

int mmssl_abi_version(void);
const char* mmssl_last_error(void);
/* 0 if the current device is compute capability 9.x (H100); fails loudly otherwise. */
int mmssl_device_check(void);
/* 1 if the row kernels (SpMM, row ops, losses) and the projection are built for embedding width d: 32, 64, 96, 128, 192
 * or 256.  The tensor-core InfoNCE (d in {64, 128}), the fused id fusion (d in {64, 128}) and the hot-row / staged-gather
 * SpMM variants (d in {64, 128, 256}) cover fewer widths; mmssl_spmm_csr_f32 at d = 32, 96, 192 takes impl 0, 4 or 16. */
int mmssl_embed_width_supported(int d);

/* ------------------------------------------------------------------ graph preparation
 * Replaces the per-call coalesce + COO->CSR conversion ATen performs inside torch.sparse.mm
 * (Models.py:69-73, :203-208) and restates the graph normalisation of main.py:89-103. */
int64_t mmssl_csr_workspace_bytes(int64_t nnz, int64_t n_rows);
/* COO (int64 row/col, fp32 values; unsorted and duplicate coordinates allowed) -> CSR sorted by
 * (row, col), stable for duplicates.  transpose != 0 builds the CSR of A^T (n_rows/n_cols are
 * then those of A^T). */
int mmssl_csr_from_coo(const int64_t* rows, const int64_t* cols, const float* vals, int64_t nnz,
                       int64_t n_rows, int64_t n_cols, int transpose, int32_t* rowptr, int32_t* colidx,
                       float* out_vals, void* workspace, int64_t workspace_bytes, void* stream);
/* vals[e] *= (rowsum + 1e-8)^-1/2  -- csr_norm(mean_flag=True), main.py:89-103 */
int mmssl_csr_row_normalize(const int32_t* rowptr, int64_t n_rows, float* vals, void* stream);

/* Where mmssl_spmm_plan cuts rows (tuning / test knob; applies to plans built afterwards, call before the *_cap functions):
 * rows above split_threshold non-zeros become segments of seg_len (deterministic ordered reduction), rows above heavy_threshold
 * segments of heavy_seg_len accumulated with vector atomics. */
int mmssl_spmm_plan_set_cuts(int split_threshold, int seg_len, int heavy_threshold, int heavy_seg_len);
/* nnz-balanced work plan: rows longer than 64 non-zeros are cut into 32-nnz segments (64-nnz for rows over
 * 1024, which accumulate atomically) that different lane groups process concurrently. */
int64_t mmssl_spmm_plan_items_cap(int64_t n_rows, int64_t nnz);
int64_t mmssl_spmm_plan_splits_cap(int64_t nnz);
int64_t mmssl_spmm_plan_segs_cap(int64_t nnz);
int64_t mmssl_spmm_plan_workspace_bytes(int64_t n_rows);
int mmssl_spmm_plan(const int32_t* rowptr, int64_t n_rows, int64_t nnz, int32_t* items4 /*[items_cap][4]*/,
                    int64_t items_cap, int32_t* split_table4 /*[splits_cap][4]*/, int32_t* counters /*[splits_cap]*/,
                    int64_t splits_cap, int32_t* totals3, void* workspace, int64_t workspace_bytes, void* stream);

/* host descriptor of a prepared sparse operand */
typedef struct {
    const int32_t* rowptr; /* [n_rows+1] */
    const int32_t* colidx; /* [nnz] */
    const float* vals;     /* [nnz] */
    int64_t n_rows, n_cols, nnz;
    const int32_t* items; /* work plan, [n_items][4] = {row, begin, end, split or -1}; row<0 = unused */
    int64_t n_items;      /* capacity actually launched over */
    const int32_t* split_table; /* [n_split_rows][4] = {first partial slot, #segments, segment length, 0} */
    int32_t* counters;
    int64_t segs_cap; /* partial-sum slots the plan may use */
} mmssl_csr_t;

/* ------------------------------------------------------------------ SpMM (the propagation operator)
 * Y_r = epi( A * X_r [+ alpha * C_r] ),   optional S_r (+)= Y_r.
 * Replaces MMSSL.mm / torch.sparse.mm (Models.py:69-73,177-186) and torch.mm(sparse,dense)
 * (Models.py:203-208) incl. the row softmax of the last layer (Models.py:203-204), the layer sum of
 * Models.py:213-214 and, with the CSR of A^T, the transposed products autograd derives. */
#define MMSSL_EPI_NONE 0
#define MMSSL_EPI_SOFTMAX 1     /* y = softmax_d(v) */
#define MMSSL_EPI_SOFTMAX_BWD 2 /* y = ysaved * (v - <v, ysaved>) */
typedef struct {
    const float* x; int64_t ldx;
    float* y; int64_t ldy;
    const float* c; int64_t ldc;           /* optional; may alias y */
    const float* ysaved; int64_t ldysaved; /* MMSSL_EPI_SOFTMAX_BWD only */
    float* s; int64_t lds;                 /* optional running sum */
    const float* sbase; int64_t ldsbase;   /* s_mode 2: S = sbase + y */
    /* fused all-gather (row-sharded tables, SURVEY 8e): where the output rows go
     *   0: y (local);  1: y is an NVSwitch MULTICAST address -> one multimem.st per 16 bytes lands in every
     *   GPU's table;  2: additionally stored to the n_peers peer-mapped tables y_peers[] over NVLink. */
    int32_t y_mode; int32_t n_peers;
    float* y_peers[8];
} mmssl_spmm_rhs_t;
/* d in {64,128,256}; nrhs in 1..3 (all right-hand sides share A and d).  s_mode: 0 none, 1 S += y, 2 S = sbase + y.
 * `partials` = zero-initialised scratch for split rows, >= a->segs_cap * nrhs * d floats (left clean by the kernel).
 * impl: 0 = automatic launch policy (128-thread blocks under 2M edges, register-capped variant above); otherwise a bit
 * set of tuning variants of the gather kernel: 2 = 8-lane groups at d = 64, 4 = 128-thread blocks, 8 = twice the
 * gathers in flight, 16 = registers capped for 6 resident blocks/SM (8|16 = both with 4 blocks/SM). */
int mmssl_spmm_csr_f32(const mmssl_csr_t* a /*host*/, int d, int nrhs, const mmssl_spmm_rhs_t* rhs /*host*/,
                       int epilogue, float alpha, int s_mode, float* partials, int64_t partials_floats, int impl, void* stream);
/* Tuning / test knob of the software-pipelined small-graph variant (impl bit 9 = 512, spmm.cu): the grid size in blocks of 128
 * threads; 0 (default) = as many as one device holds at once.  Every lane group walks items g, g + groups, g + 2 groups, ... */
int mmssl_spmm_pipe_set_blocks(int blocks);

/* TMA-staged variant for large power-law graphs: the X rows of the `n_hot` highest-degree columns
 * (hot_ids, by decreasing degree) are staged once per CTA into shared memory with cp.async.bulk and
 * gathers of those columns are served from shared memory.  colidx_hot = a->colidx with hot columns
 * encoded as -(slot+1).  Same contract / epilogues as mmssl_spmm_csr_f32. */
int mmssl_spmm_hot_f32(const mmssl_csr_t* a /*host*/, const int32_t* colidx_hot, const int32_t* hot_ids, int n_hot, int d,
                       int nrhs, const mmssl_spmm_rhs_t* rhs /*host*/, int epilogue, float alpha, int s_mode,
                       float* partials, int64_t partials_floats, void* stream);

/* Staged-gather pipeline (spmm_bulk.cu; north_star: "stages neighbour embeddings through TMA into shared memory with
 * warp-shuffle partial sums"): one warp per BUCKET of <= 32 consecutive non-zeros / <= 8 whole rows (or one 32-chunk of a longer
 * row); every neighbour row of the bucket and the row-indexed epilogue operands travel as asynchronous copies into the warp's
 * shared-memory slots (warp-wide 16-byte cp.async, or one cp.async.bulk per row completed on an mbarrier: variant bit 16), no
 * register holds a row in flight.  Same contract / epilogues as mmssl_spmm_csr_f32 for nrhs <= 2 (not: softmax-backward
 * together with a running sum).  `a` carries the operand's CSR arrays and the BUCKET plan's split_table / counters / segs_cap
 * (`items` is not used), `partials` >= a->segs_cap * nrhs * d zeroed floats.
 * variant: bits 4-7 warps per block (0 = 4), bits 8-15 buckets per warp (0 auto), bit 16 TMA copy engine. */
int64_t mmssl_spmm_bulk_plan_splits_cap(int64_t nnz);
int64_t mmssl_spmm_bulk_plan_segs_cap(int64_t nnz);
int64_t mmssl_spmm_bulk_plan_buckets_cap(int64_t n_rows, int64_t nnz);
int64_t mmssl_spmm_bulk_plan_workspace_bytes(int64_t n_rows);
/* buckets8[k] = {first row, #rows, first position, #positions, split-row index or -1, chunk index, 0, 0}; entries beyond
 * totals3[0] stay zero (0 rows: skipped by the kernel).  totals3 = {#buckets, #split rows, #partial slots}. */
int mmssl_spmm_bulk_plan(const int32_t* rowptr, int64_t n_rows, int64_t nnz, int32_t* split_table4, int32_t* counters,
                         int64_t splits_cap, int32_t* buckets8 /*[buckets_cap][8]*/, int64_t buckets_cap, int32_t* totals3,
                         void* workspace, int64_t workspace_bytes, void* stream);
int mmssl_spmm_bulk_f32(const mmssl_csr_t* a /*host*/, const int32_t* buckets8, int64_t n_buckets, int d, int nrhs,
                        const mmssl_spmm_rhs_t* rhs /*host*/, int epilogue, float alpha, int s_mode, float* partials,
                        int64_t partials_floats, int variant, void* stream);

/* Second half of a row-sharded product computed as partial products (rowshard_step.py, schedule "reduce_scatter"): the rank's
 * rows of the SUM over all ranks' partial tables -- rhs[r].x = multicast address of the rank's first row (multicast != 0:
 * multimem.ld_reduce, the NVSwitch adds the replicas) or a local pointer to reduced rows (multicast == 0) -- followed by the
 * SpMM epilogue of mmssl_spmm_csr_f32 (+ alpha*C, softmax / softmax backward, store, running sum; same rhs fields). */
int mmssl_reduce_rows_epilogue(int64_t n_rows, int d, int nrhs, const mmssl_spmm_rhs_t* rhs /*host*/, int epilogue, float alpha,
                               int s_mode, int multicast, void* stream);

/* ------------------------------------------------------------------ dense fp32 GEMM (CUDA-core path)
 * C = alpha * op(A) * op(B) + beta * C, row-major.  Used for the d x d "attention" mixing
 * (Models.py:139-169 == v * sum_h Wcat[h], SURVEY appendix B.1) and as the verification path of the
 * projection.  split_k > 1 accumulates with float atomics (C must hold beta*C already; beta is then ignored). */
int mmssl_sgemm(int trans_a, int trans_b, int64_t m, int64_t n, int64_t k, float alpha, const float* a, int64_t lda,
                const float* b, int64_t ldb, float beta, float* c, int64_t ldc, int split_k, void* stream);

/* ------------------------------------------------------------------ projection (wgmma + TMA)
 * X = F * W^T + b  and  dW = dX^T * F, fp32 semantics via a bf16 hi/lo split (3 MMAs per product),
 * replaces nn.Linear image_trans/text_trans forward and weight gradient (Models.py:28-31,173-174).
 * Declared in the "projection" section below once built (mmssl_proj_*). */

/* ------------------------------------------------------------------ row-wise fused glue
 * out = e + rate * z / max(||z||, 1e-12)          (Models.py:196-197)
 * zn = normalised z (contiguous [n,d]), nrm[n] = ||z|| */
int mmssl_id_fuse_fwd(const float* z, int64_t ldz, const float* e, int64_t lde, int64_t n, int d, float rate,
                      float* out, int64_t ldo, float* zn, float* nrm, void* stream);
/* dz = rate * d(normalize)(g)   (backward of the above w.r.t. z; the gradient w.r.t. e is g itself) */
int mmssl_id_fuse_bwd(const float* g, int64_t ldg, const float* zn, const float* nrm, int64_t n, int d, float rate,
                      float* dz, int64_t lddz, void* stream);
/* Fused id fusion (Models.py:139-169 closed form + :188-197), d in {64,128}:
 *   wsum[d][d] = sum_h wcat[h*d:(h+1)*d][:]
 *   fwd: m = coef*(ya [+ yb]); z = m*wsum; out = e + rate*z/max(|z|,1e-12); zn, nrm saved
 *   bwd (takes wsum_t): dz = rate*d(normalize)(g); out_a = coef*dz*wsum^T + ext_a (+ ext_b when out_b is NULL), out_b likewise;
 *        dw_part[block][d*d] = per-block partial of m^T dz  (mmssl_id_fuse2_blocks(n) blocks)
 *   dwcat[h] = sum of all partial tiles, for every head h */
int mmssl_wsum(const float* wcat, int d, int heads, float* wsum, float* wsum_t /* transposed copy */, void* stream);
int mmssl_id_fuse2_blocks(int64_t n);
int mmssl_id_fuse2_fwd(const float* ya, int64_t lda, const float* yb, int64_t ldb, float coef, const float* wsum,
                       const float* e, int64_t lde, int64_t n, int d, float rate, float* out, int64_t ldo, float* zn,
                       float* nrm, void* stream);
int mmssl_id_fuse2_bwd(const float* g, int64_t ldg, const float* zn, const float* nrm, const float* ya, int64_t lda,
                       const float* yb, int64_t ldb, float coef, const float* wsum_t, int64_t n, int d, float rate,
                       const float* ext_a, int64_t ldea, const float* ext_b, int64_t ldeb, float* out_a, int64_t ldoa,
                       float* out_b, int64_t ldob, float* dw_part, void* stream);
int mmssl_dwcat_reduce(const float* part_u, int nu, const float* part_i, int ni, int d, int heads, float* dwcat,
                       void* stream);
/* out = s * inv_layers + rate * (normalize(a) + normalize(b))   (Models.py:213-218)
 * sumsq_partials[blocks] receives per-block sum(a^2 + b^2) (feeds feat_reg, main.py:252-257). */
int mmssl_combine_fwd(const float* s, int64_t lds, const float* a, int64_t lda, const float* b, int64_t ldb, int64_t n,
                      int d, float inv_layers, float rate, float* out, int64_t ldo, float* sumsq_partials,
                      int64_t n_partials, void* stream);
int64_t mmssl_combine_partials(int64_t n, int d);
/* ga = ga_ext + rate * d(normalize)(a; g) + reg_coef * a   (and the same for b); ga_ext may be NULL */
int mmssl_combine_bwd(const float* g, int64_t ldg, const float* a, int64_t lda, const float* b, int64_t ldb,
                      const float* ga_ext, int64_t ldgae, const float* gb_ext, int64_t ldgbe, int64_t n, int d,
                      float rate, float reg_coef, float* ga, int64_t ldga, float* gb, int64_t ldgb, void* stream);
/* t = y * (alpha*g - <alpha*g, y>)  (softmax backward for one tensor) */
int mmssl_softmax_bwd(const float* y, int64_t ldy, const float* g, int64_t ldg, int64_t n, int d, float alpha,
                      float* t, int64_t ldt, void* stream);
/* y = alpha * (alpha_dev ? *alpha_dev : 1) * x + beta * y, strided rows (alpha_dev: optional device scalar) */
int mmssl_axpby(const float* x, int64_t ldx, int64_t n, int d, float alpha, const float* alpha_dev, float beta, float* y, int64_t ldy, void* stream);
/* dropout apply: y = x * mask (mask holds 0 or 1/(1-p)) ; mask may be NULL (copy) */
int mmssl_mul_mask(const float* x, int64_t ldx, const float* mask, int64_t ldm, int64_t n, int d, float* y, int64_t ldy, void* stream);
/* per-block sums of squares of an [n,d] matrix: partials[mmssl_sumsq_blocks(n,d)] */
int64_t mmssl_sumsq_blocks(int64_t n, int d);
int mmssl_sumsq(const float* x, int64_t ldx, int64_t n, int d, float* partials, void* stream);

/* ------------------------------------------------------------------ BPR   (main.py:368-371, :499-511)
 * rows: u = UF[users[k]], p = IF[pos[k]], n = IF[neg[k]]  (index arrays may be NULL = identity).
 * mode bit 0: write per-block partial sums  part[2*b] = sum softplus(-(u.p-u.n)),  part[2*b+1] = sum (|u|^2+|p|^2+|n|^2)/2
 * mode bit 1: accumulate gradients  (atomic adds when indices are given, plain adds otherwise):
 *     d/du = -sigmoid(-x)*(p-n)*w_mf + w_reg*u, ...  with w_mf = g_mf/B, w_reg = g_emb*reg_coef,
 *     g_mf / g_emb read from device scalars (NULL = 1.0). */
int64_t mmssl_bpr_blocks(int64_t batch, int d);
int mmssl_bpr(const float* uf, int64_t ldu, const float* itf, int64_t ldi, const float* itf_neg, int64_t ldin,
              const int64_t* users, const int64_t* pos, const int64_t* neg, int64_t batch, int d, int mode,
              float reg_coef, const float* g_mf, const float* g_emb, float* part, float* g_uf, int64_t ldgu,
              float* g_pos, int64_t ldgp, float* g_neg, int64_t ldgn, void* stream);

/* ------------------------------------------------------------------ InfoNCE  (main.py:211-249)
 * loss = mean_i -log( B_ii / (sum_j R_ij + sum_j B_ij - R_ii) + 1e-8 ),  R = exp(a a^T/tau), B = exp(a b^T/tau),
 * a = normalize(z1[idx]), b = normalize(z2[idx]).  Work buffers are caller-provided:
 *   a,b [n,d]; na,nb [n]; stats [4*n + 2*n*ceil(n/64)] ; coef [2*n]; ga,gb [n,d] (zeroed by prepare). */
int mmssl_infonce_prepare(const float* z1, int64_t ldz1, const float* z2, int64_t ldz2, const int64_t* idx, int64_t n,
                          int d, float* a, float* b, float* na, float* nb, float* ga, float* gb, void* stream);
int64_t mmssl_infonce_stats_floats(int64_t n);
int64_t mmssl_infonce_loss_blocks(int64_t n);
/* row statistics + per-row loss partials (loss_part[mmssl_infonce_loss_blocks(n)] = block sums of loss_i)
 * and backward coefficients coef[2n] scaled by g_loss (device scalar, NULL = 1) / n. */
int mmssl_infonce_stats(const float* a, const float* b, int64_t n, int d, float inv_tau, float* stats, float* coef,
                        const float* g_loss, float* loss_part, void* stream);
int mmssl_infonce_grad(const float* a, const float* b, int64_t n, int d, float inv_tau, const float* coef, float* ga,
                       float* gb, void* stream);
/* through the normalisation, then (atomic) scatter-add into the tables: g_z1[idx[i]] += ..., g_z2[idx[i]] += ... */
/* Tensor-core InfoNCE for n <= 2048, d in {64, 128} (loss_tc.cu): the similarity tiles a a^T, a b^T on wgmma (bf16 hi/lo, three
 * MMAs per product), exp / row sums / diagonal in the register epilogue, the exponentials kept as bf16 hi/lo matrices in `workspace`;
 * the backward = three split-K wgmma products of those matrices with [a | u.a], b, u.a + one combine kernel.  Same inputs and
 * outputs as mmssl_infonce_stats / mmssl_infonce_grad (ga, gb are WRITTEN here, accumulated there). */
int mmssl_infonce_tc_supported(int64_t n, int d);
int64_t mmssl_infonce_tc_workspace_bytes(int64_t n, int d);
int mmssl_infonce_stats_tc(const float* a, const float* b, int64_t n, int d, float inv_tau, float* stats, float* coef,
                           const float* g_loss, float* loss_part, void* workspace, int64_t workspace_bytes, void* stream);
/* prepare (gather + normalise, as mmssl_infonce_prepare) + operand split + statistics in one call */
int mmssl_infonce_forward_tc(const float* z1, int64_t ldz1, const float* z2, int64_t ldz2, const int64_t* idx, int64_t n, int d,
                             float inv_tau, float* a, float* b, float* na, float* nb, float* stats, float* coef, const float* g_loss,
                             float* loss_part, void* workspace, int64_t workspace_bytes, void* stream);
/* phase: -1 all on `stream`; 0 operands, 1..3 the three products (independent of each other), 4 combine */
int mmssl_infonce_grad_tc(const float* a, const float* b, int64_t n, int d, float inv_tau, const float* coef, const float* stats,
                          float* ga, float* gb, void* workspace, int64_t workspace_bytes, int phase, void* stream);
int mmssl_infonce_scatter(const float* ga, const float* gb, const float* a, const float* b, const float* na,
                          const float* nb, const int64_t* idx, int64_t n, int d, float* g_z1, int64_t ldg1, float* g_z2,
                          int64_t ldg2, void* stream);

/* ------------------------------------------------------------------ loss assembly  (main.py:420 without the GAN term)
 * out[0]=total, [1]=mf, [2]=emb, [3]=feat_reg, [4]=cl.  Sums the partial arrays in index order (deterministic).
 * total = mf + emb + feat + cl_rate*cl ; mf = sum(bpr_part[2b])/batch ; emb = reg_coef*sum(bpr_part[2b+1]) ;
 * feat = feat_coef * (sum fr_u + sum fr_i) ; cl = cl_mult * (sum nce1)/n_nce + (sum nce2)/n_nce  */
int mmssl_loss_assemble(const float* bpr_part, int64_t n_bpr_blocks, int64_t batch, float reg_coef, const float* fr_u,
                        int64_t n_fr_u, const float* fr_i, int64_t n_fr_i, float feat_coef, const float* nce1,
                        int64_t n_nce1, const float* nce2, int64_t n_nce2, int64_t n_nce_rows, float cl_rate,
                        float* out5, void* stream);

/* ------------------------------------------------------------------ AdamW  (main.py:76-80, :427-429; torch.optim.AdamW semantics)
 * Up to 16 tensors per call.  *step_dev (device int32) is the 1-based step number to use (see mmssl_step_tick). */
#define MMSSL_ADAMW_MAX_TENSORS 16
int mmssl_step_tick(int32_t* step_dev, void* stream);
int mmssl_adamw(int n_tensors, float* const* p /*host array of device ptrs*/, const float* const* g, float* const* m,
                float* const* v, const int64_t* numel /*host*/, const int32_t* step_dev, float lr, float beta1,
                float beta2, float eps, float weight_decay, void* stream);

/* Data-parallel optimiser step fused with its collectives over NVSwitch multicast (one kernel): this rank's slice
 * [begin, begin+count) of the flat buckets: g = multimem.ld_reduce(add) over all ranks' gradient buckets * inv_world,
 * AdamW with slice-local m, v (indexed from 0), new parameters multimem.st'ed into every rank's parameter bucket.
 * p_mc / g_mc are the multicast addresses of the symmetric parameter / gradient buckets, p_local this rank's copy.
 * The caller barriers all ranks before and after.  step is 1-based (host value). */
int mmssl_dp_fused_adamw(const float* p_local, float* p_mc, const float* g_mc, float* m, float* v, int64_t begin,
                         int64_t count, float inv_world, int step, float lr, float beta1, float beta2, float eps,
                         float weight_decay, void* stream);
/* the same with the 1-based step number read from device memory (mmssl_step_tick): the launch is CUDA-graph capturable */
int mmssl_dp_fused_adamw_dev(const float* p_local, float* p_mc, const float* g_mc, float* m, float* v, int64_t begin,
                             int64_t count, float inv_world, const int32_t* step_dev, float lr, float beta1, float beta2,
                             float eps, float weight_decay, void* stream);

/* ------------------------------------------------------------------ GPU triple sampler (SURVEY 8f "next" #1)
 * Semantics of Data.sample (utility/load_data.py:153-191): `batch` distinct users with >= 1
 * training item (with replacement only if batch > n_exist), one uniform positive from the user's CSR row
 * (indptr/indices int64, rows sorted), one uniform negative rejected against the row.  Counter-based RNG
 * keyed by (seed, step); step is read from *step_dev when non-NULL (graph replay), else step_host.
 * mmssl_sample_triples: batch <= 1024, one CTA; claim[n_exist] is a work table initialised once with
 * mmssl_sampler_init and left clean by every launch. */
int mmssl_sampler_init(int32_t* claim, int64_t n_exist, void* stream);
int mmssl_sample_triples(const int64_t* indptr, const int64_t* indices, const int64_t* exist, int64_t n_exist,
                         int64_t n_items, int batch, uint64_t seed, const int32_t* step_dev, int32_t step_host,
                         int32_t* claim, int64_t* users, int64_t* pos, int64_t* neg, void* stream);
/* Any batch size: the users are the slots of the `batch` smallest keys (hash32(seed, step, slot) << 32 | slot), found by a
 * multi-CTA radix select over all n_exist slots (O(n_exist) per call) and returned in key order; batch == n_exist is a
 * permutation.  batch > n_exist draws with replacement.  Depends only on (seed, step, batch).  The workspace
 * (mmssl_sampler_workspace_bytes, 0 when batch > n_exist) is zero-filled once before its first use and left so by every
 * call; no allocation and no host synchronisation per call, so the launch is CUDA-graph capturable.  The workspace holds
 * the select's counters between kernels: calls that share one workspace must not overlap (one stream, or one graph
 * replay at a time); concurrent callers use one workspace each. */
int64_t mmssl_sampler_workspace_bytes(int64_t n_exist, int batch);
int mmssl_sample_triples_multi(const int64_t* indptr, const int64_t* indices, const int64_t* exist, int64_t n_exist,
                               int64_t n_items, int batch, uint64_t seed, const int32_t* step_dev, int32_t step_host,
                               void* workspace, int64_t workspace_bytes, int64_t* users, int64_t* pos, int64_t* neg,
                               void* stream);

/* ------------------------------------------------------------------ evaluation (SURVEY 8f "next" #3)
 * Trainer.test -> test_torch / test_one_user (main.py:301-306, utility/batch_test.py:21-36, :83-169) and
 * utility/metrics.py:9-19, :43-90, fused: scores of users[n_eval] against all items are ranked on the fly (no
 * [users x items] matrix in HBM), training items (CSR rows, int64, SORTED) are skipped, the max(Ks) best remain,
 * equal scores keep the lower item id first (heapq.nlargest over ascending ids).  Outputs:
 *   ranked[n_eval, kmax] item ids best first (-1 past the end of a short list); ranked_scores (may be NULL);
 *   hits[n_eval, kmax] 1/0 membership in the held-out row (CSR, SORTED), -1 past the end (may be NULL);
 *   per_user[n_eval, 4, n_ks] fp64 = precision, recall, ndcg, hit_ratio at every K (reference quirks kept:
 *   ideal DCG from the retrieved hit list, precision divisor shrinks with short lists, recall / len(held-out));
 *   scores_out[n_eval, n_items] (may be NULL; debugging / tests).  ks_host is a HOST array of n_ks cut-offs;
 *   mmssl_eval_rank / _full take 1..8 cut-offs in 1..64, mmssl_eval_rank_wide any number of cut-offs in 1..2^26.
 *   kmax = max(Ks); the hit list has min(kmax, #non-training items) entries.
 * mmssl_eval_reduce: result[m] = mean over users of per_user[:, m] (batch_test.py:159-163), fixed order, any n_metrics. */
int mmssl_eval_rank(const float* user_emb, int64_t ldu, const float* item_emb, int64_t ldi, int64_t n_items, int d,
                    const int64_t* users, int64_t n_eval, const int64_t* train_indptr, const int64_t* train_indices,
                    const int64_t* held_indptr, const int64_t* held_indices, const int32_t* ks_host, int n_ks,
                    int32_t* ranked, float* ranked_scores, int32_t* hits, double* per_user, float* scores_out,
                    void* stream);
/* Full mode (--test_flag full, batch_test.py:38-68, metrics.py:95-100): the same ranking outputs as mmssl_eval_rank,
 * plus auc_per_user[n_eval] fp64 = roc_auc_score over the user's non-training items in [0, n_items), positives =
 * distinct held-out ids among them, ties counted 1/2.  Reference quirks kept: NaN when there is one class only, 0 when
 * the user has no candidate item or a candidate's score is NaN / inf.  Exact from integer pair counts.
 * Workspace: users whose held-out row is longer than mmssl_eval_full_stage() keep their positives' keys in
 * pos_ws[pos_ws_off[g] ...], a slot of next_pow2(row length) uint32; pos_ws_off[n_eval] is read only for those users
 * (pos_ws may be NULL when there is none). */
int mmssl_eval_full_stage(void);
int mmssl_eval_rank_full(const float* user_emb, int64_t ldu, const float* item_emb, int64_t ldi, int64_t n_items, int d,
                         const int64_t* users, int64_t n_eval, const int64_t* train_indptr, const int64_t* train_indices,
                         const int64_t* held_indptr, const int64_t* held_indices, const int32_t* ks_host, int n_ks,
                         int32_t* ranked, float* ranked_scores, int32_t* hits, double* per_user, float* scores_out,
                         double* auc_per_user, uint32_t* pos_ws, const int64_t* pos_ws_off, void* stream);
/* Wide path: the same outputs for any Ks (more than 8 cut-offs, K > 64, K > n_items).  ks_host (validation, sizing) and
 * ks_dev (read by the kernel) hold the same n_ks cut-offs.  auc_per_user == NULL: part mode; else full mode with
 * pos_ws / pos_ws_off as in mmssl_eval_rank_full.  Per-user candidate buffers hold cap = 2 ksel + 256 (rounded up to 128)
 * keys, ksel = min(kmax, n_items): in shared memory while a CTA's 8 buffers and user vectors fit in 112 KiB, else in
 * key_ws, which must hold mmssl_eval_wide_workspace_bytes(n_eval, kmax, n_items, d) bytes (0 in the shared-memory case):
 * one slot of 8 cap keys per CTA, at most 528 slots and at most 512 MiB (at least one slot). */
int64_t mmssl_eval_wide_workspace_bytes(int64_t n_eval, int kmax, int64_t n_items, int d);
int mmssl_eval_rank_wide(const float* user_emb, int64_t ldu, const float* item_emb, int64_t ldi, int64_t n_items, int d,
                         const int64_t* users, int64_t n_eval, const int64_t* train_indptr, const int64_t* train_indices,
                         const int64_t* held_indptr, const int64_t* held_indices, const int32_t* ks_host, const int32_t* ks_dev,
                         int n_ks, int32_t* ranked, float* ranked_scores, int32_t* hits, double* per_user, float* scores_out,
                         double* auc_per_user, uint32_t* pos_ws, const int64_t* pos_ws_off, uint64_t* key_ws, void* stream);
int mmssl_eval_reduce(const double* per_user, int64_t n_eval, int n_metrics, double* result, void* stream);

/* ------------------------------------------------------------------ GAN side (SURVEY 8f "next" #2), see csrc/gan.cu
 * Device ops sequenced by mmssl_b200/gan.py; the Discriminator of Models.py:224-245 on n rows (LeakyReLU(True) is the
 * identity and does not appear), gradient_penalty main.py:140-160, u_sim_calculation main.py:283-298, the real rows of
 * main.py:348-351.  All matrices fp32 row-major and CONTIGUOUS ([n][h]); h need not be a multiple of 4.
 * Specification of every op: the function of the same name in tests/gan_ops_cpu.py.
 *   bn_fwd      training-mode BatchNorm1d of (a + bias) then the dropout mask: h_out, ah (normalised), rstd; running stats
 *               updated in place (momentum 0.1, unbiased variance)
 *   bn_bwd      dy = dh*mask, dgamma, dbeta, da (gradient w.r.t. the Linear output in front)
 *   gp_rev_bn   adjoint of bn_bwd seeded with q = adjoint(da): adjoint(dh), adjoint(ah), adjoint(rstd), gamma gradient
 *   bn_fwd_rev  adjoint of bn_fwd given adjoint(h) and the extra adjoints of ah / rstd: adjoint(a), gamma / beta gradients
 *   head_fwd    s = sigmoid(h2 . w3 + b3), s_sum = sum(s)            (D output = 100 s)
 *   head_bwd    backward of sum(coef * 100 s): dh2, dz, dw3, db3
 *   gp_rows     gp = lam * mean_i (||gx_i|| - 1)^2 and gbar = d gp / d gx      (sq_scratch: n floats)
 *   gp_head_rev adjoint of head_bwd + head_fwd: adjoint(h2) of the forward, w3 / b3 gradients (z_bar_scratch: n floats)
 *   usim_finish y = rows of `scores` with the user's training items (CSR, int64) zeroed, L2-normalised; nrm = the norms
 *   usim_bwd_pre d_raw = (g - y <g,y>) / nrm, zero at the training items
 *   real_rows   normalize(softmax(R_row - log_log_scale * log(-log(u + 1e-8) + 1e-8) / tau) + pre_scale * ui_sim) */
int mmssl_gan_bn_fwd(const float* a, const float* bias, const float* gamma, const float* beta, const float* mask,
                     float* running_mean, float* running_var, int64_t n, int64_t h, float* h_out, float* ah, float* rstd,
                     void* stream);
int mmssl_gan_bn_bwd(const float* dh, const float* mask, const float* gamma, const float* ah, const float* rstd, int64_t n,
                     int64_t h, float* da, float* dy, float* dgamma, float* dbeta, void* stream);
int mmssl_gan_gp_rev_bn(const float* q, const float* dy, const float* ah, const float* rstd, const float* gamma,
                        const float* mask, int64_t n, int64_t h, float* dh_bar, float* ah_bar, float* r_bar, float* g_gamma,
                        void* stream);
int mmssl_gan_bn_fwd_rev(const float* h_bar, const float* mask, const float* gamma, const float* ah, const float* rstd,
                         const float* ah_bar, const float* r_bar, int64_t n, int64_t h, float* a_bar, float* g_gamma,
                         float* g_beta, void* stream);
int mmssl_gan_colsum(const float* x, int64_t n, int64_t h, float* out, void* stream);
int mmssl_gan_head_fwd(const float* h2, const float* w3, const float* b3, int64_t n, int64_t h, float* s, float* s_sum,
                       void* stream);
int mmssl_gan_head_bwd(const float* s, float coef, const float* w3, const float* h2, int64_t n, int64_t h, float* dh2,
                       float* dz, float* dw3, float* db3, void* stream);
int mmssl_gan_gp_rows(const float* gx, int64_t n, int64_t w, float lam, float* gbar, float* sq_scratch, float* gp,
                      void* stream);
int mmssl_gan_gp_head_rev(const float* dh2_bar, const float* dz, const float* s, const float* w3, const float* h2,
                          int64_t n, int64_t h, float* z_bar_scratch, float* h_bar, float* g_w3, float* g_b3, void* stream);
int mmssl_gan_usim_finish(const float* scores, const int64_t* users, const int64_t* indptr, const int64_t* indices,
                          int64_t rows, int64_t w, float* y, float* nrm, void* stream);
int mmssl_gan_usim_bwd_pre(const float* g, const float* y, const float* nrm, const int64_t* users, const int64_t* indptr,
                           const int64_t* indices, int64_t rows, int64_t w, float* d_raw, void* stream);
int mmssl_gan_real_rows(const int64_t* users, const int64_t* indptr, const int64_t* indices, const float* uniform,
                        const float* ui_sim, int64_t rows, int64_t w, float log_log_scale, float tau, float pre_scale,
                        float* out, void* stream);
/* out = alpha[row] * xr + (1 - alpha[row]) * xf ;  acc += alpha * x (flat) ;  row gather / atomic row scatter-add */
int mmssl_gan_interpolate(const float* alpha, const float* xr, const float* xf, int64_t rows, int64_t w, float* out,
                          void* stream);
int mmssl_gan_add_scaled(float* acc, const float* x, float alpha, int64_t total, void* stream);
int mmssl_gan_gather_rows(const float* table, int64_t ld, const int64_t* rows, int64_t n_rows, int d, float* out,
                          void* stream);
int mmssl_gan_scatter_add_rows(float* table, int64_t ld, const int64_t* rows, int64_t n_rows, int d, const float* src,
                               void* stream);

/* ------------------------------------------------------------------ row-sharded hot step (shard.cu, SURVEY 8e)
 * A rank holds the rows [lo, hi) of a table; the batch indexes the FULL table (main.py:368-370, :411-412).
 * mmssl_gather_owned: out[j] = table_local[idx[j] - lo] when the rank owns row idx[j], zeros otherwise (summing the
 *   ranks' outputs gives the batch rows everywhere).  mmssl_scatter_add_owned: table_local[idx[j] - lo] += src[j] for the
 *   owned rows only (atomic; duplicate ids accumulate). */
int mmssl_gather_owned(const float* table, int64_t ld, const int64_t* idx, int64_t lo, int64_t hi, int64_t n, int d, float* out,
                       int64_t ldo, void* stream);
int mmssl_scatter_add_owned(float* table, int64_t ld, const int64_t* idx, int64_t lo, int64_t hi, int64_t n, int d,
                            const float* src, int64_t lds, void* stream);
/* All-gather without NCCL: this rank's rows src[rows, d] are stored at dst (+ the same offset in every peer table):
 * y_mode 1: dst is the NVSwitch MULTICAST address of the rank's row block in a symmetric table (one multimem.st per 16 bytes,
 * replicated into every GPU's copy, the local one included); y_mode 2: dst is the local block, peers[n_peers] (host array) the
 * peer-mapped addresses of the same block on the other GPUs; y_mode 0: plain local copy.  Same store paths as the SpMM epilogue. */
int mmssl_publish_rows(const float* src, int64_t lds, int64_t rows, int d, float* dst, int64_t ldd, int y_mode, int n_peers,
                       float* const* peers, void* stream);
/* All-reduce(sum) without NCCL: dst[0..n) = sum over the ranks' copies of a symmetric buffer, read through its multicast address
 * (multimem.ld_reduce, the switch adds the replicas).  The caller barriers all ranks before (contributions written) and after. */
int mmssl_mc_allreduce_sum(const float* src_mc, float* dst, int64_t n, void* stream);

/* ------------------------------------------------------------------ modality-graph bookkeeping of the full step (regraph.cu)
 * mmssl_topk_rows: ids[rows, k] (int64) = columns of the k largest entries of every row of x[rows, w], best first, equal
 *   values keep the lower column first -- torch.topk(G_*_u_sim_detach, int(n_items * m_topk_rate)) at main.py:397,400.
 * mmssl_pair_append: x[j] = users[j % batch], y[j] = ids.flat[j] for j < batch * k -- the python lists of main.py:398-402
 *   (the x list tiles the user vector k times, the y list is row-major: the reference's pairing, kept).
 * mmssl_degree_values: vals[j] = (deg(idx[j]) + 1e-8)^-1/2 with deg = number of entries carrying the same index --
 *   csr_norm(mean_flag=True) (main.py:89-103) applied to the 0/1 (duplicates summed) matrix of main.py:379-391, per COO
 *   entry; deg_scratch holds n_rows int32. */
int mmssl_topk_rows(const float* x, int64_t ldx, int64_t rows, int64_t w, int k, int64_t* ids, void* stream);
int mmssl_pair_append(const int64_t* users, int64_t batch, const int64_t* ids, int k, int64_t* x, int64_t* y, void* stream);
int mmssl_degree_values(const int64_t* idx, int64_t n, int64_t n_rows, int32_t* deg_scratch, float* vals, void* stream);

/* ------------------------------------------------------------------ projection (wgmma + TMA), see proj_tc.cu */
int mmssl_split_bf16(const float* x, int64_t ldx, int64_t rows, int64_t cols, uint16_t* hi, uint16_t* lo, int64_t ldo,
                     void* stream);
/* transposed split: hi/lo [cols][ldo] from x [rows][cols] (optionally multiplied by mask [rows][cols]) */
int mmssl_split_bf16_t(const float* x, int64_t ldx, const float* mask, int64_t ldm, int64_t rows, int64_t cols,
                       uint16_t* hi, uint16_t* lo, int64_t ldo, void* stream);
/* the same + colsum[c] = sum_r (x * mask)[r][c]   (db of the projection's backward, Models.py:173-174, from the tile pass) */
int mmssl_split_bf16_t_colsum(const float* x, int64_t ldx, const float* mask, int64_t ldm, int64_t rows, int64_t cols,
                              uint16_t* hi, uint16_t* lo, int64_t ldo, float* colsum, void* stream);
int64_t mmssl_gemm_bf16x3_workspace_floats(int64_t m, int64_t n, int64_t k, int* split_k_out);
/* partial[s][m][n] (fp32) = sum over the s-th K slice of (Ahi+Alo)[m,k] * (Bhi+Blo)[n,k]  (lo*lo dropped).
 * A: [m][lda] bf16 K-major, B: [n][ldb] bf16 K-major; n in {64,128,256}. */
int mmssl_gemm_bf16x3(const uint16_t* a_hi, const uint16_t* a_lo, int64_t lda, const uint16_t* b_hi,
                      const uint16_t* b_lo, int64_t ldb, int64_t m, int64_t n, int64_t k, int split_k, float* partial,
                      void* stream);
/* One problem of a grouped projection GEMM: the operands and result of mmssl_gemm_bf16x3. */
typedef struct {
    const uint16_t* a_hi;
    const uint16_t* a_lo;
    int64_t lda;
    const uint16_t* b_hi;
    const uint16_t* b_lo;
    int64_t ldb;
    int64_t m, n, k;
    float* partial;   /* [split_k][m][n] */
    int32_t split_k;
    int32_t reserved;
} mmssl_gemm_problem_t;
/* Plan of a group of one or two problems (mnk = m0, n0, k0, m1, n1, k1; the same n): per problem the split count and the
 * partial-buffer size in floats; optionally the units in the order the CTAs walk them, 4 int32 each
 * (problem, m_tile, kb_begin, kb_end), at most units_cap of them.  max_ctas caps the grid (0 = one resident wave) and must
 * be the value later passed to mmssl_gemm_bf16x3_group.  Returns the number of units, or -1 on bad arguments. */
int64_t mmssl_gemm_bf16x3_group_plan(int n_problems, const int64_t* mnk, int max_ctas, int* split_out, int64_t* floats_out,
                                     int32_t* units_out, int64_t units_cap);
/* Every problem's partial[s][m][n] as mmssl_gemm_bf16x3 with the same split_k would write it, in ONE persistent launch. */
int mmssl_gemm_bf16x3_group(int n_problems, const mmssl_gemm_problem_t* problems, int max_ctas, void* stream);
/* General-width variant for the GAN side (gemm_wide.cu): c[m][ldc] = alpha * (Ahi+Alo)[m,k] * (Bhi+Blo)[n,k]^T (+ c when
 * accumulate != 0), any n >= 1, no split-K, alpha / accumulate applied in the epilogue; replaces the Discriminator's
 * nn.Linear products and their closed-form backward / gradient-penalty variants (Models.py:224-245, main.py:140-160). */
int mmssl_gemm_bf16x3_wide(const uint16_t* a_hi, const uint16_t* a_lo, int64_t lda, const uint16_t* b_hi,
                           const uint16_t* b_lo, int64_t ldb, int64_t m, int64_t n, int64_t k, float alpha, int accumulate,
                           float* c, int64_t ldc, void* stream);
/* Tuning / test knob of the kernel above: k-blocks (64 of K each) chained into one accumulator before the epilogue folds
 * the pass into C with fp32 adds (default 16 = 1024 of K; bounds the tensor core's accumulation error, gemm_wide.cu). */
int mmssl_gemm_wide_set_chunk(int k_blocks);
/* y[m][ldy + col_off] = (sum_s partial[s][m][n] + bias[n]) * mask[m][n]     (bias / mask may be NULL) */
int mmssl_proj_epilogue(const float* partial, int split_k, int64_t m, int64_t n, const float* bias, const float* mask,
                        int64_t ldm, float* y, int64_t ldy, float* y_pre, int64_t ldyp, void* stream);
/* dw[n][ldw] (+)= sum_s partial[s][m][n]^T  (m = feature dim, n = embed dim) */
int mmssl_wgrad_epilogue(const float* partial, int split_k, int64_t m, int64_t n, float* dw, int64_t ldw, int accumulate,
                         void* stream);
/* column sums: db[n] (+)= sum_rows (g * mask)[rows][n] */
int mmssl_colsum(const float* g, int64_t ldg, const float* mask, int64_t ldm, int64_t rows, int n, float* out,
                 int accumulate, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MMSSL_B200_H */
