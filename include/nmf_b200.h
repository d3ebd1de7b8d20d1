/*
 * nmf_b200.h -- C ABI of the H100-native multiplicative-update NMF engine (libnmf_b200.so).
 *
 * This is the drop-in boundary for ONE hot path of yoyololicon/pytorch-NMF (torchnmf 0.3.5):
 * the body of BaseComponent.fit()'s iteration loop for dense targets
 *
 *     torchnmf/nmf.py:366-407   for n_iter in range(max_iter): W update, H update, loss every 10th
 *
 * i.e. reconstruct (nmf.py:691-693 NMF, :776-779 NMFD) + _double_backward_update (nmf.py:52-92)
 * + the KL denominators (nmf.py:122-131) + metrics.beta_div (metrics.py:60-96).  The reference has
 * no FFI: its seam is Python.  The binding a maintainer adds on the reference side is
 * the ctypes stub shown in INTEGRATION.md; the Python host side shipped here
 * (pytorch-nmf_b200/torchnmf_b200) is that stub plus the unchanged NMF/NMFD module surface.
 *
 * Conventions
 *   - plain C: pointers, sizes, doubles.  No torch / C++ types.
 *   - all matrix pointers are DEVICE pointers to fp32, row-major, reference layout, except that a dense target V may also
 *     hold fp16 or bf16 elements (nmfb200_nmf_set_target / nmfb200_nmfd_set_target: read where they are, no fp32 copy):
 *       NMF : V (N,C)   W (C,R)   H (N,R)            V ~= H @ W^T            (nmf.py:659-662)
 *       NMFD: V (B,C,L) W (C,R,T) H (B,R,L-T+1)      V ~= conv1d(H, flip(W)) (nmf.py:743-750)
 *   - a context holds one model, NMF or NMFD (NMF2D / NMF3D included), fixed by its create call.  The nmfb200_nmf_* and
 *     nmfb200_nmfd_* calls take only contexts of their model (NMFB200_ERR_INVALID, "wrong context kind", otherwise); the
 *     calls without a model in their name serve both.  A batched context (nmfb200_nmf_batched_create,
 *     nmfb200_nmfnd_batched_create) holds many problems of one model; its own calls are named after their kind.
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream).  Every call is
 *     asynchronous on that stream unless documented as synchronising.
 *   - W / H are the caller's storages (the nn.Parameter .data of the reference); updates are
 *     performed IN PLACE on them (nmf.py:92).  V is borrowed read-only.
 *   - every function returns 0 on success; on failure a non-zero code, and
 *     nmfb200_last_error() describes it.  There is no CPU fallback anywhere in this library.
 */
#ifndef NMF_B200_H_
#define NMF_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 2: the update / loss / raw-terms / W-apply / sync calls serve both models under one name, and both dense set_target
 * calls take the target's element type */
#define NMFB200_ABI_VERSION 2

/* arithmetic mode of the contraction kernels */
enum {
  NMFB200_PREC_AUTO      = -1, /* f16 tensor-core path when the rank allows it (R <= 128), else f32 */
  NMFB200_PREC_F32       = 0,  /* fused CUDA-core kernels, fp32 operands and accumulators (exact), any rank */
  NMFB200_PREC_F16       = 1,  /* wgmma, fp16 operands, fp32 accumulate                           */
  NMFB200_PREC_F16_SPLIT = 2   /* wgmma, fp16 hi/lo split factors (~22-bit), fp16 ratio tile      */
};

/* element type of a dense target V (nmfb200_nmf_set_target / nmfb200_nmfd_set_target).  The kernels convert each element
 * to fp32 where they load it; fp16 and bf16 values are exact in fp32, so a half-precision target gives the results, bit for
 * bit, of the same values registered as fp32. */
enum {
  NMFB200_DTYPE_F32  = 0,
  NMFB200_DTYPE_F16  = 1,      /* IEEE binary16 (__half)        */
  NMFB200_DTYPE_BF16 = 2       /* bfloat16 (__nv_bfloat16)      */
};

/* error codes */
enum {
  NMFB200_OK = 0,
  NMFB200_ERR_INVALID = 1,     /* bad argument / unsupported shape for the requested mode */
  NMFB200_ERR_CUDA = 2,        /* CUDA runtime / driver error                             */
  NMFB200_ERR_STATE = 3        /* call order violated (e.g. update before set_target)     */
};

typedef struct nmfb200_ctx nmfb200_ctx;

int         nmfb200_abi_version(void);
const char* nmfb200_last_error(void);
/* "src=<sha256/16 of csrc/* + this header> nvcc=<version> arch=sm_90a built=<date time>": which sources this binary is */
const char* nmfb200_build_info(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
int64_t     nmfb200_launch_count(void);

/* Synchronises `stream` and reports whether any kernel of this library aborted an internal wait (a protocol bug or a
 * wedged device), on the context's device: 0 = healthy, non-zero = the results since the last check are invalid.  The
 * caller's current device is left unchanged, as it is by every entry point that takes a context. */
int nmfb200_ctx_check_health(nmfb200_ctx* ctx, void* stream);

/* ---- dense NMF ------------------------------------------------------------------------- */

/* Allocate the engine workspace for an (N,C) target of rank R on CUDA device `device`.
 * Mirrors the sizes fixed by NMF.__init__ (nmf.py:679-689).  Any rank 1 <= R <= 65535 x 256 runs on the fp32 kernels
 * (above 256 components in blocks of 256, each recomputing the reconstruction tile); the tensor-core precisions need
 * R <= 128, and a sparse target (nmfb200_nmf_set_target_sparse) R <= 256. */
int nmfb200_nmf_create(nmfb200_ctx** out, int device, int64_t N, int64_t C, int64_t R, int precision);
void nmfb200_destroy(nmfb200_ctx* ctx);
/* which NMFB200_PREC_* the context resolved to */
int nmfb200_precision(const nmfb200_ctx* ctx);
/* which NMFB200_PREC_* the contraction kernels use for this beta (the tensor-core path covers beta != 2 for
 * rank <= 64 and beta == 1 for rank <= 128; everything else runs the fp32 kernels) */
int nmfb200_precision_for_beta(const nmfb200_ctx* ctx, double beta);

/* Register the target V: device elements of type `dtype` (NMFB200_DTYPE_*), leading dimension ldv >= C.  Builds the
 * engine-private operand copies and the V-only loss terms.  Replaces nothing in the reference: V is simply the argument of
 * fit() (nmf.py:299).  V stays borrowed: every later call of this context (update_*, iterate, loss, loss_prefetch_w,
 * raw_terms, contract_only, update_w_peer, target_minmax) reads it.  NMFB200_ERR_INVALID for an unknown dtype or a V not
 * aligned to its element size (2 bytes for fp16 / bf16, 4 for fp32); no other alignment is required.  Asynchronous. */
int nmfb200_nmf_set_target(nmfb200_ctx* ctx, const void* V, int64_t ldv, int dtype, void* stream);
/* min / max of the registered target (fit()'s validation, nmf.py:329-336).  Synchronises. */
int nmfb200_target_minmax(nmfb200_ctx* ctx, float* vmin, float* vmax, void* stream);

/* n_iter consecutive MU iterations with both factors trainable: exactly n_iter x (update_w; update_h), i.e.
 * nmf.py:366-391 repeated, in one host call. */
int nmfb200_nmf_iterate(nmfb200_ctx* ctx, float* W, float* H, double beta, double gamma, double l1_reg,
                        double l2_reg, int n_iter, void* stream);
/* nmfb200_loss, evaluated at the factors the NEXT W update starts from (nmf.py:393-402 runs right before nmf.py:367 of the
 * following iteration): on the tensor-core path for beta == 1 the loss sums come out of the W update's own contraction pass
 * (one lg2 per element on the S tile that pass forms anyway, instead of a pass over V of its own), and the next
 * nmfb200_update_w / nmfb200_nmf_iterate on UNCHANGED factors with the same beta skips its contraction.  Any other
 * call in between (or a stop of the fit) simply discards the prefetched numerators.  Elsewhere: identical to
 * nmfb200_loss. */
int nmfb200_nmf_loss_prefetch_w(nmfb200_ctx* ctx, const float* W, const float* H, double beta,
                                double* loss_dev, void* stream);

/* ---- batched NMF: many independent problems of one shape in one context ---------------------------------- */

/* A context for B independent NMF problems of one shape, on the fp32 CUDA-core kernels: problem b has the target V_b (N,C)
 * and the factors W_b (C,R) = W + b C R and H_b (N,R) = H + b N R of the caller's (B,C,R) / (B,N,R) storages.  Every
 * update, loss and column-sum launch runs all B problems at once, in the number of launches one problem takes, and each
 * problem keeps the tile plan and summation order of a single-problem NMFB200_PREC_F32 context of (N, C, R): its factors
 * and loss are, bit for bit, those of that context.  Workspace: B times the partial slabs, column sums and loss partials of
 * one such context.  NMFB200_ERR_INVALID for B < 1, R > 256, or a batch too large for the launch grids.
 * On a batched context: nmfb200_update_w / _update_h / nmfb200_nmf_iterate / nmfb200_sync_factors serve it;
 * nmfb200_loss writes B doubles (loss_dev[b]); nmfb200_raw_terms returns [B N_f R numerators | B R column sums (beta 1) or
 * B N_f R denominators] (N_f: the rows of the updated factor), and nmfb200_raw_terms_numel reports that length;
 * nmfb200_target_minmax covers every problem; nmfb200_precision_for_beta reports NMFB200_PREC_F32.  nmfb200_set_mask,
 * nmfb200_set_weight, nmfb200_w_apply, nmfb200_nmf_set_target and its sparse / observed forms, nmfb200_nmf_loss_prefetch_w,
 * nmfb200_nmf_contract_only, nmfb200_nmf_cd_update / _iterate and the peer calls return NMFB200_ERR_INVALID.  The three
 * calls below and nmfb200_nmf_batched_cd_update / _iterate take batched contexts only (NMFB200_ERR_INVALID otherwise). */
int nmfb200_nmf_batched_create(nmfb200_ctx** out, int device, int64_t B, int64_t N, int64_t C, int64_t R);
/* A batch of B problems of different row counts over one C: problem b has lengths[b] (1 <= lengths[b] <= N; `lengths` is B
 * host int64, read during the call) rows, stored in the same padded layouts as a nmfb200_nmf_batched_create context's --
 * V_b's first lengths[b] rows, W_b (C,R) = W + b C R, H_b's first lengths[b] rows of H + b N R.  Every call that serves a
 * batched NMF context serves it, with these differences:
 *   - problem b runs, bit for bit, the plan of a single NMFB200_PREC_F32 context of (lengths[b], C, R): its own contraction
 *     chunks, loss chunks and column-sum blocks, each launch holding every problem's blocks on grid x;
 *   - no call reads rows lengths[b].. of V_b or H_b, and no call writes them (nor those rows of nmfb200_raw_terms' output);
 *   - nmfb200_target_minmax covers every problem's first lengths[b] rows (of a shared target too);
 *   - nmfb200_plca_iterate and nmfb200_plca_loss serve it: problem b is the PLCA problem of V_b's first lengths[b] rows, W_b,
 *     H_b's first lengths[b] rows and Z_b, bit for bit that of a nmfb200_nmf_batched_create context of (1, lengths[b], C, R);
 *     rows lengths[b].. of H_b, Hz_b, H_alpha_b and of the raw H numerators in `work` are neither read nor written;
 *   - nmfb200_nmf_batched_cd_update / _iterate return NMFB200_ERR_INVALID.
 * Workspace: the sum over the problems of a single context's partial slabs, column-sum and loss partials, not B times the
 * largest.  NMFB200_ERR_INVALID, before any device work, for B < 1, R > 256, a null `lengths`, a length outside [1, N], and
 * a launch whose problems' blocks together pass grid x (2^31 - 1) or whose loss partials pass 2^31. */
int nmfb200_nmf_batched_create_ragged(nmfb200_ctx** out, int device, int64_t B, int64_t N, int64_t C, int64_t R,
                                      const int64_t* lengths);
/* Register the targets: problem b reads V + b batch_stride, rows ldv >= C elements apart, elements of type `dtype`.
 * batch_stride 0: one V shared by every problem (restarts of one fit); otherwise batch_stride >= N ldv.  Alignment and dtype
 * checks as nmfb200_nmf_set_target.  V stays borrowed.  Asynchronous. */
int nmfb200_nmf_batched_set_target(nmfb200_ctx* ctx, const void* V, int64_t ldv, int64_t batch_stride, int dtype,
                                   void* stream);
/* Which problems run from now on: `active` is B device bytes, borrowed (read by every later launch), null = every problem.
 * A problem flagged 0 is skipped by every update, loss and raw-terms launch: its factors, its loss_dev slot and its
 * raw-terms slots are left as they are, at the cost of one flag read per block. */
int nmfb200_nmf_batched_set_active(nmfb200_ctx* ctx, const uint8_t* active, void* stream);

/* Sparse target for beta 1 and beta 2 (nmf.py:603-638 `_nmf_sp_recon_beta_pos_neg`, :95-119): registers V (N x C) in both
 * compressed forms -- CSR (crow[N+1], col[nnz], val[nnz]) and CSC = CSR of V^T (ccol[C+1], row[nnz], val_t[nnz]) -- int64
 * indices, fp32 values, device pointers borrowed until the next set_target*.  v_norm_kl / v_norm_eu: `_get_V_norm` nmf.py:161-170
 * for beta 1 / 2.  update_w / update_h / iterate / loss then evaluate the update terms at the non-zeros only (one warp per row
 * or column, fp32) and never form the dense product; any other beta returns NMFB200_ERR_INVALID (densify the target), as
 * does a context of rank R > 256. */
int nmfb200_nmf_set_target_sparse(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow, const int64_t* col, const float* val,
                                  const int64_t* ccol, const int64_t* row, const float* val_t,
                                  double v_norm_kl, double v_norm_eu, void* stream);
/* The same registration (same arguments and meaning, same refusals), on a context that then serves every beta > 0 without
 * densifying V.  Beta 1 and 2 run exactly the kernels above.  Any other beta (x = w_c . h_n + eps, nmf.py:621-636):
 *   numerators at the non-zeros only (num_H[n,:] = sum_{c in row n} v x^(beta-2) W[c,:], the W side over the columns);
 *   denominators over all N x C cells but V-free (den_H[n,:] = sum_c x^(beta-1) W[c,:]): the fp32 contraction without the V
 *   tile and the numerator GEMM, on the dense fp32 plan, so they equal a dense fp32 context's bit for bit;
 *   loss = V_norm + sum_all x^beta / beta - sum_nnz v x^(beta-1) / (beta-1), V_norm = sum_nnz v^beta / (beta (beta-1)) taken
 *   in the loss launch itself (v_norm_kl / v_norm_eu serve beta 1 / 2 only).
 * Device memory stays O(nnz + (N + C) R).  beta <= 0 returns NMFB200_ERR_INVALID.  Every other set_target* on the context
 * turns this off again. */
int nmfb200_nmf_set_target_sparse_any_beta(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow, const int64_t* col,
                                           const float* val, const int64_t* ccol, const int64_t* row, const float* val_t,
                                           double v_norm_kl, double v_norm_eu, void* stream);
/* Fit only the OBSERVED cells of V, listed as sparse entries: the nnz stored entries of the two compressed forms (layout and
 * borrowing as nmfb200_nmf_set_target_sparse) are exactly the observed cells, each once, and val / val_t hold V's value
 * there (zeros allowed: an observed zero is a cell of the loss, not a missing one).  No v_norm: the loss takes V's terms per
 * cell.  From then on the context fits beta_div(WH[obs], V[obs]) at every beta, as nmfb200_set_mask does on a dense target,
 * with every update nmf.py:78-92 applied to the two backward passes of that loss (x = w_c . h_n):
 *   num_H[n,:] = sum_{c observed in row n} v a(x) W[c,:]      den_H[n,:] = sum_{c observed in row n} b(x) W[c,:]
 *   (beta 2: a = 1, b = x; beta 1: a = 1 / (x + eps), b = 1; other: a = (x + eps)^(beta-2), b = (x + eps)^(beta-1)),
 * the W side over the columns; both from ONE gather per row or column (one warp each, fp32, in stored order: no atomics),
 * O(nnz R) per update, no dense product, Gram matrix or column sum.  update_w, update_h, nmf_iterate, loss,
 * nmf_loss_prefetch_w (= loss), raw_terms (raw_terms_numel: 2 x the factor's numel at every beta), w_apply and
 * target_minmax (the observed values; +inf / -inf when nnz == 0) follow it.  precision_for_beta reports NMFB200_PREC_F32,
 * nmf_peer_supported 0; contract_only returns NMFB200_ERR_STATE and set_mask NMFB200_ERR_INVALID, as on a sparse context;
 * a context of rank R > 256 returns NMFB200_ERR_INVALID.  Any other set_target* turns the mode off again.  Asynchronous. */
int nmfb200_nmf_set_target_observed(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow, const int64_t* col,
                                    const float* val, const int64_t* ccol, const int64_t* row, const float* val_t,
                                    void* stream);
/* The same as nmfb200_nmf_set_target_observed, plus one fp32 weight per stored entry: wt in the order of val (CSR), wt_t in
 * the order of val_t (CSC), device pointers borrowed like the rest (null only when nnz == 0, else NMFB200_ERR_INVALID).  The
 * context then fits sum_obs w d_beta(v | x): each entry's terms in both gathers are multiplied by its weight,
 *   num_H[n,:] = sum_c (w v) a(x) W[c,:]      den_H[n,:] = sum_c (w b(x)) W[c,:]      loss = sum_obs w loss_term,
 * so at beta 1 den = the weighted rows of the other factor.  The weights should be positive and finite (an entry of weight 0
 * is better left out).  Everything else -- the calls that follow it, the refusals, what turns it off -- is
 * nmfb200_nmf_set_target_observed's.  Asynchronous. */
int nmfb200_nmf_set_target_observed_weighted(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow, const int64_t* col,
                                             const float* val, const int64_t* ccol, const int64_t* row, const float* val_t,
                                             const float* wt, const float* wt_t, void* stream);

/* Row-sharded W update over PEER MEMORY (ranks of one NVLink domain, one process per GPU, 2..8 ranks) -- the fused form of
 * raw_terms(which = 0) -> all-reduce -> w_apply below, without a collective library call on the data path:
 *   local contraction -> a pack kernel that pushes this rank's partial [C*R | R] into its slot of EVERY rank's exchange block
 *   (posted NVLink writes) and publishes its iteration counter -> ONE ratio-stage kernel per rank that waits for all counters,
 *   sums the slots of its own block in rank order (the replicas of W stay bit-identical) and applies nmf.py:78-92.
 * Setup (once per context, collective): peer_alloc returns this rank's 64-byte CUDA IPC handle; exchange the handles (any
 * transport; the Python host side uses torch.distributed); peer_connect takes all `world` handles in rank order.  Then every
 * rank calls update_w_peer for every W update.  peer_supported: 1 if this context / beta can use it (tensor-core path,
 * rank % 4 == 0, beta != 2).  A rank that never arrives makes the kernel give up after ~2 s; nmfb200_ctx_check_health reports it. */
int nmfb200_nmf_peer_supported(const nmfb200_ctx* ctx, double beta);
int nmfb200_nmf_peer_alloc(nmfb200_ctx* ctx, void* ipc_handle_out /* 64 bytes */);
int nmfb200_nmf_peer_connect(nmfb200_ctx* ctx, int world, int rank, const void* ipc_handles /* world x 64 bytes */);
int nmfb200_nmf_peer_world(const nmfb200_ctx* ctx);          /* connected ranks, 0 if none */
int nmfb200_nmf_peer_release(nmfb200_ctx* ctx);
int nmfb200_nmf_update_w_peer(nmfb200_ctx* ctx, float* W, const float* H,
                              double beta, double gamma, double l1_reg, double l2_reg, void* stream);

/* Profiling aid for bench.py's roofline line: launches ONLY the fused contraction kernel of the W update
 * (which = 0) or the H update (which = 1) into the engine's scratch, leaving W and H untouched. */
int nmfb200_nmf_contract_only(nmfb200_ctx* ctx, const float* W, const float* H, int which, double beta,
                              void* stream);

/* Coordinate descent at beta 2 (HALS, sklearn's solver="cd"): one update of W (which = 0) or H (which = 1) in place, that
 * minimises 1/2 |V - H W^T|^2 + l1_reg (sum W + sum H) + l2_reg / 2 (|W|^2 + |H|^2) over that factor by one sweep over its
 * columns.  With X the updated factor, A = V^T H (W) or V W (H) and B = the other factor's Gram matrix, both formed once at
 * the start of the update, for k = 0 .. R-1 in order and every row c:
 *   X[c,k] <- max(0, X[c,k] + (A[c,k] - sum_j X[c,j] B[j,k] - l1_reg - l2_reg X[c,k]) / (B[k,k] + l2_reg)),
 * X[c,j] already updated for j < k; a column with B[k,k] + l2_reg == 0 is left as it is.  The floor is exactly 0, and a
 * later multiplicative update cannot move an entry that is exactly 0.  A is, bit for bit, nmfb200_raw_terms(which, 2.0)'s
 * numerator: on a dense target the fp32 contraction without S = W H^T (any target dtype and row stride), on a sparse one
 * (nmfb200_nmf_set_target_sparse / _sparse_any_beta) the gather at the stored entries.  B comes from the fixed-order Gram
 * kernel of the sparse beta-2 path, and each row's sweep sums in an order fixed by R alone: the result is deterministic.
 * Dense contexts of any precision run on these fp32 kernels and mark the tensor-core operand copies of X stale.  The Gram
 * scratch (2 R^2 floats and the Gram kernel's block partials) is allocated at the first call on a dense context.
 * NMFB200_ERR_INVALID for NMFD / NMF2D / NMF3D, batched and observed-cell contexts, a context with a mask or a weight, and
 * R > 256; NMFB200_ERR_STATE before set_target.  Asynchronous. */
int nmfb200_nmf_cd_update(nmfb200_ctx* ctx, float* W, float* H, int which, double l1_reg, double l2_reg, void* stream);
/* n_iter x (nmfb200_nmf_cd_update of W; of H with the new W) in one host call; same contexts and refusals. */
int nmfb200_nmf_cd_iterate(nmfb200_ctx* ctx, float* W, float* H, double l1_reg, double l2_reg, int n_iter, void* stream);
/* The same update on a nmfb200_nmf_batched_create context, for every active problem (nmfb200_nmf_batched_set_active) in
 * the launches one problem takes (four per factor update, whatever B): problem b's W_b / H_b (W + b C R, H + b N R) are,
 * bit for bit, what nmfb200_nmf_cd_update gives on a single NMFB200_PREC_F32 context of (N, C, R) with target V_b -- each
 * problem keeps that context's contraction chunks, Gram plan and summation orders.  An inactive problem's factors are not
 * written.  Workspace: the A partials use the context's partial slabs; the Gram scratch, allocated at the first call, is
 * B (2 R^2 + max(nb(N), nb(C)) R^2) floats, nb(rows) the Gram blocks of nmfb200_nmf_sparse_plan (at most 128).
 * NMFB200_ERR_INVALID for any other context kind (a single dense or sparse NMF, an observed-cell, NMFD or batched NMFD
 * context), a null context or pointer, which not 0 / 1, and for B x ceil(max(N, C) / 32) sweep blocks (or B x the Gram
 * blocks) past grid x (2^31 - 1); NMFB200_ERR_STATE before nmfb200_nmf_batched_set_target.  Asynchronous. */
int nmfb200_nmf_batched_cd_update(nmfb200_ctx* ctx, float* W, float* H, int which, double l1_reg, double l2_reg,
                                  void* stream);
/* n_iter x (nmfb200_nmf_batched_cd_update of W; of H with the new W) in one host call; n_iter < 0 and the refusals above
 * return NMFB200_ERR_INVALID. */
int nmfb200_nmf_batched_cd_iterate(nmfb200_ctx* ctx, float* W, float* H, double l1_reg, double l2_reg, int n_iter,
                                   void* stream);
/* Coordinate descent at beta 2 on the observed cells (CCD++, Yu et al. 2012, made non-negative), on a context whose target
 * was set by nmfb200_nmf_set_target_observed or _observed_weighted.  One update of W (which = 0) or H (which = 1) in place
 * minimises  1/2 sum_{(n,c) observed} w (v - h_n . w_c)^2 + l1_reg (sum W + sum H) + l2_reg / 2 (|W|^2 + |H|^2)  over that
 * factor (w = 1 without weights) by one exact sweep over its columns.  Every row s of the updated factor X runs on its own,
 * over the observed cells O_s of its segment (a column of V for W, a row for H), with f_j the other factor's row of cell j
 * and r = v - f_j . x_s at the current x_s; for k = 0 .. R-1 in order:
 *   num = sum_{j in O_s} w_j r_j f_{j,k},  hess = sum_{j in O_s} w_j f_{j,k}^2 + l2_reg,
 *   if hess != 0:  x_{s,k} <- max(0, x_{s,k} + (num - l1_reg - l2_reg x_{s,k}) / hess),
 * entries j < k already updated.  The floor is exactly 0; a row with no observed cell and l2_reg = 0 is left as it is.
 * With every cell observed and unit weights this is nmfb200_nmf_cd_update's update in exact arithmetic.  One warp per
 * segment sums in the segment's stored order: no atomics, the result is deterministic.  O(observed x R) work per update,
 * in ceil(R / 32) passes over the observed entries; above rank 32 a residual workspace of one float per observed entry is
 * allocated at the first call.  These are separate calls: nmfb200_nmf_cd_update / _iterate still refuse observed-cell
 * contexts.  NMFB200_ERR_STATE before any set_target*; NMFB200_ERR_INVALID for any other target form (dense, with or
 * without a mask or weight, or sparse), NMFD / NMF2D / NMF3D and batched contexts, a null context or pointer, and which
 * not 0 / 1.  Asynchronous. */
int nmfb200_nmf_observed_cd_update(nmfb200_ctx* ctx, float* W, float* H, int which, double l1_reg, double l2_reg,
                                   void* stream);
/* n_iter x (nmfb200_nmf_observed_cd_update of W; of H with the new W) in one host call; n_iter < 0 and the refusals above
 * return NMFB200_ERR_INVALID. */
int nmfb200_nmf_observed_cd_iterate(nmfb200_ctx* ctx, float* W, float* H, double l1_reg, double l2_reg, int n_iter,
                                    void* stream);

/* ---- NMFD (1-D convolutive NMF), NMF2D, NMF3D ------------------------------------------------ */

/* Sizes as NMFD.__init__ (nmf.py:762-774) with ndim = 1: V (B,C,L), W (C,R,T), H (B,R,L-T+1), vdims = {L}, kdims = {T}.
 * NMF2D / NMF3D (nmf.py:782-865, :868-942: conv2d / conv3d with flipped kernels and full padding) are the same context type
 * with ndim = 2 or 3 convolved axes: vdims = the target's sizes over those axes, kdims = kernel_size; V (B,C,*vdims),
 * W (C,R,*kdims), H (B,R,*(vdims - kdims + 1)), all contiguous.  Every NMFD call serves all three.  With ndim 2 or 3,
 * precision auto or f32 runs the fp32 kernels; NMFB200_PREC_F16 runs beta 1 on the tensor-core sliding GEMMs of NMFD, over
 * the outer axes too (R <= 256 and the limits of nmfb200_nmfnd_tc_plan, whose message create returns otherwise), and every
 * other beta on the fp32 kernels, as an NMFD context at f16 does (nmfb200_precision_for_beta says which). */
int nmfb200_nmfnd_create(nmfb200_ctx** out, int device, int64_t B, int64_t C, int ndim, const int64_t* vdims,
                         int64_t R, const int64_t* kdims, int precision);
/* Register a contiguous target of element type `dtype` (NMFB200_DTYPE_*), with the checks of nmfb200_nmf_set_target. */
int nmfb200_nmfd_set_target(nmfb200_ctx* ctx, const void* V, int dtype, void* stream);

/* ---- batched NMFD / NMF2D / NMF3D: many independent problems of one shape in one context ---------------------------- */

/* A context for P independent NMFD / NMF2D / NMF3D problems of one shape, on the fp32 CUDA-core kernels.  Each problem has
 * the shape of nmfb200_nmfnd_create(B, C, ndim, vdims, R, kdims) (the same checks apply to it): problem p has the target
 * V_p (B,C,*vdims) and the factors W_p = W + p C R prod(kdims) and H_p = H + p B R prod(vdims - kdims + 1) of the caller's
 * (P,C,R,*kdims) / (P,B,R,*(vdims - kdims + 1)) storages; its B clips share W_p.  Every reconstruction, wgrad, dgrad,
 * column-sum and ratio-stage launch runs all P problems at once (grid z of the sliding kernels holds P x B lines, problem
 * after problem; grid z of wgrad P x its splits, in launches of at most 65535), and each problem keeps the plan and
 * summation order of a single NMFB200_PREC_F32 context of its shape: the same wgrad / dgrad splits, tiles and loss blocks,
 * so its factors and loss are, bit for bit, that context's.  Workspace: P times the fp32 NMFD context's -- the ratio tile Pn
 * (and Pp at beta != 1) of V's size, the split partial slabs, the column sums and the loss partials.
 * NMFB200_ERR_INVALID, naming the limit, for P < 1, P x B >= 2^31 (the kernels' line index), P x loss partials per problem
 * >= 2^31, P x column-sum blocks past grid x, or P x B x C x prod(vdims) > 2^46.
 * On a batched NMFD context: nmfb200_update_w / _update_h / nmfb200_sync_factors serve it; nmfb200_loss writes P doubles
 * (loss_dev[p]); nmfb200_raw_terms returns [P x factor numerators | P R column sums (beta 1) or P x factor denominators],
 * nmfb200_raw_terms_numel reports that length; nmfb200_target_minmax covers every problem; nmfb200_precision_for_beta
 * reports NMFB200_PREC_F32.  nmfb200_set_mask, nmfb200_set_weight, nmfb200_w_apply, nmfb200_nmfd_set_target and every
 * nmfb200_nmf_* call return NMFB200_ERR_INVALID.  The two calls below take batched NMFD contexts only. */
int nmfb200_nmfnd_batched_create(nmfb200_ctx** out, int device, int64_t P, int64_t B, int64_t C, int ndim,
                                 const int64_t* vdims, int64_t R, const int64_t* kdims);
/* A batch of P problems of different lengths along the LAST convolved axis (the sliding axis): problem p has lengths[p]
 * (T <= lengths[p] <= L, T = kdims[ndim - 1] and L = vdims[ndim - 1]; `lengths` is P host int64, read during the call)
 * positions there, stored in the same padded layouts as a nmfb200_nmfnd_batched_create context's of vdims -- V_p's first
 * lengths[p] positions of every line of the last axis, W_p as there, and H_p's first lengths[p] - T + 1 positions of every
 * line of its last axis (L - T + 1 long).  Every call that serves a batched NMFD context serves it, with these differences:
 *   - problem p runs, bit for bit, the plan of a single NMFB200_PREC_F32 context of (B, C, vdims with the last size
 *     lengths[p], R, kdims): its own reconstruction grid and loss blocks, dgrad splits and column-sum blocking, each launch
 *     sized for the largest problem, a problem's surplus blocks exiting at once;
 *   - no call reads positions lengths[p].. of V_p or lengths[p] - T + 1.. of H_p, and no call writes the latter (nor those
 *     positions of nmfb200_raw_terms' output);
 *   - nmfb200_target_minmax covers every problem's real positions (of a shared target too);
 *   - nmfb200_plca_iterate and nmfb200_plca_loss return NMFB200_ERR_INVALID.
 * Workspace: the sum over the problems of a single context's ratio tiles, split partial slabs, column-sum and loss
 * partials, not P times the largest.  NMFB200_ERR_INVALID, before any device work, for whatever
 * nmfb200_nmfnd_batched_create refuses at the padded shape, a null `lengths`, a length outside [T, L], and P x B x R
 * past grid x (2^31 - 1). */
int nmfb200_nmfnd_batched_create_ragged(nmfb200_ctx** out, int device, int64_t P, int64_t B, int64_t C, int ndim,
                                        const int64_t* vdims, int64_t R, const int64_t* kdims, const int64_t* lengths);
/* Register the targets: problem p reads the contiguous block V + p problem_stride of B C prod(vdims) elements of type
 * `dtype`.  problem_stride 0: one V shared by every problem (restarts of one fit); otherwise problem_stride >=
 * B C prod(vdims).  Checks as nmfb200_nmfd_set_target; the min / max run over every problem.  V stays borrowed.
 * Asynchronous. */
int nmfb200_nmfd_batched_set_target(nmfb200_ctx* ctx, const void* V, int64_t problem_stride, int dtype, void* stream);
/* Which problems run from now on, with the contract of nmfb200_nmf_batched_set_active: `active` is P device bytes, borrowed,
 * null = every problem; a problem flagged 0 is skipped by every launch (its factors, loss_dev slot and raw-terms slots are
 * left as they are) at the cost of one flag read per block. */
int nmfb200_nmfd_batched_set_active(nmfb200_ctx* ctx, const uint8_t* active, void* stream);

/* ---- batched PLCA / SIPLCA / SIPLCA2 / SIPLCA3: the EM iteration on a batched NMF or NMFD context ------------------ */

/* Each problem p of a batched NMF context (PLCA) or batched NMFD context (SIPLCA, SIPLCA2, SIPLCA3) is one PLCA problem on
 * the normalised target V_p / sum(V_p): W (P,C,R,*kdims), H (P,N,R) or (P,B,R,*(vdims - kdims + 1)), Z (P,R) and
 * Hz = H diag(Z) in H's shape, all contiguous fp32.  The context's factor pair is (W, Hz).  flags: which factors the EM step
 * updates (a frozen Z takes W's column sums as the prior, and with W frozen too H's own). */
#define NMFB200_PLCA_TRAIN_W 1
#define NMFB200_PLCA_TRAIN_H 2
#define NMFB200_PLCA_TRAIN_Z 4
/* Floats of the caller's `work` buffer of nmfb200_plca_iterate on this context: the raw W and H numerators of every problem
 * and the EM step's scratch.  -1 for a null or non-batched context. */
int64_t nmfb200_plca_work_numel(const nmfb200_ctx* ctx);
/* n_iter x (the raw W numerators dW, the raw H numerators dHz -- each bit for bit nmfb200_raw_terms' numerator at beta 1 --
 * then the EM step of every active problem) with no return to the host.  The EM step is the reference's plca.py:252-289 on
 * dW and dH = dHz Z (the Z from before the step): Z <- Z relu(sum H dHz), that product kept as the prior, then the alpha
 * (Z + alpha - 1, thresholded at eps) and Z / sum(Z); W <- W relu(dW) / prior (or / its column sums when Z is frozen), then
 * the alpha, threshold and renormalisation; H likewise; then Hz = H Z.  One launch per EM step, one block per problem: every
 * sum runs in an order fixed by the problem's shape, independent of P and of which problems are active.  W_alpha, H_alpha,
 * Z_alpha: null (alpha = 1) or device fp32 buffers of the factor's batched shape holding alpha.  A problem flagged inactive
 * (nmfb200_nmf_batched_set_active / nmfb200_nmfd_batched_set_active) keeps W, H, Z and Hz.  `work`: device fp32,
 * nmfb200_plca_work_numel floats.  A ragged NMF batch (nmfb200_nmf_batched_create_ragged) is served: problem b's EM step
 * runs over its first lengths[b] rows of H and Hz, every sum in the order of a batched context of (1, lengths[b], C, R), so
 * its W, Z and those rows of H and Hz equal that context's bit for bit; the padding rows are neither read nor written.
 * NMFB200_ERR_INVALID for a ragged NMFD batch (nmfb200_nmfnd_batched_create_ragged), any other context kind, rank > 256 or
 * unknown flags; NMFB200_ERR_STATE before set_target.  Asynchronous. */
int nmfb200_plca_iterate(nmfb200_ctx* ctx, float* W, float* H, float* Z, float* Hz, float* work, int flags,
                         const float* W_alpha, const float* H_alpha, const float* Z_alpha, int n_iter, void* stream);
/* loss_dev[p] (double) = kl_div(norm_p X_p, norm_p V_p) for every active problem p, X_p the reconstruction from (W, Hz) and
 * V_p the registered (normalised) target: the reference's de-normalised PLCA loss (plca.py:245,293), without materialising
 * X.  norm_dev: P device floats.  The batched KL loss launch with each problem's target and reconstructed cell scaled by
 * norm_p; an inactive problem's slot is left as it is.  A ragged NMF batch: problem b's loss over its first lengths[b] rows,
 * on its own loss plan, bit for bit the value of a batched context of (1, lengths[b], C, R); a ragged NMFD batch returns
 * NMFB200_ERR_INVALID.  Asynchronous. */
int nmfb200_plca_loss(nmfb200_ctx* ctx, const float* W, const float* Hz, const float* norm_dev, double* loss_dev,
                      void* stream);

/* ---- sparse-target PLCA (PLSA): the EM step's gradients at the stored entries only ------------------------------------ */

/* A context of its own kind for one PLCA problem on a sparse target V (N,C) with nnz stored entries, rank R
 * (1 <= R <= 65535 x 256), with the factor pair W (C,R) and Hz = H diag(Z) (N,R).  Its device workspace is
 * 4 nnz + 8 ceil(N / 8) + 8 R (nb(N) + nb(C)) bytes, nb(rows) = ceil(rows / max(256, ceil(rows / 1024))) <= 1024: the ratio
 * of each stored entry, the loss partials of the row gather and the column sums' partials, nothing of size N x C
 * (nmfb200_plca_sparse_device_bytes reports it).  Only the nmfb200_plca_sparse_* calls, nmfb200_destroy,
 * nmfb200_ctx_check_health and nmfb200_precision* (NMFB200_PREC_F32) take it; every other call that takes a context returns
 * NMFB200_ERR_INVALID ("wrong context kind").  NMFB200_ERR_INVALID for sizes below 1, nnz < 0, and ceil(max(N, C) / 8) past
 * grid x (2^31 - 1). */
int nmfb200_plca_sparse_create(nmfb200_ctx** out, int device, int64_t N, int64_t C, int64_t R, int64_t nnz);
/* Register V / sum(V) in both compressed forms: CSR (crow[N+1], col[nnz], val[nnz]: the normalised fp32 values) and CSC
 * (ccol[C+1], row[nnz]), int64 indices, each segment in ascending index order; perm[nnz] holds, for the e-th CSC entry, its
 * position in the CSR form (the entry's value is val[perm[e]]).  Device pointers, borrowed until the next set_target or
 * nmfb200_destroy.  NMFB200_ERR_INVALID for a null pointer (col, val, row and perm may be null when nnz is 0).  No device
 * work. */
int nmfb200_plca_sparse_set_target(nmfb200_ctx* ctx, const int64_t* crow, const int64_t* col, const float* val,
                                   const int64_t* ccol, const int64_t* row, const int64_t* perm, void* stream);
/* The raw gradients of one EM step (plca.py:252-253) at the current W and Hz, without touching either:
 *   P[n,c] = val / (hz_n . w_c + eps) at each stored entry,   dW = P^T Hz (C,R),   dHz = P W (N,R),
 * into `out` = [dW | dHz] (C R + N R floats), or nothing when `out` is null.  Rows and columns that store nothing get zero
 * gradients.  One gather over the CSR rows (one warp per row) forms each entry's dot product and P once and, at R <= 256,
 * accumulates dHz; one gather over the CSC columns reads P through perm and accumulates dW without a dot product.  At
 * R <= 256, dW and dHz are bit for bit the beta-1 numerators of nmfb200_raw_terms on a nmfb200_nmf_set_target_sparse
 * context holding the same values with the factor pair (W, Hz).  Above rank 256 the row gather takes the dot product over
 * blocks of 256 components and writes P, and both gradients come from gathers of P, one block of 256 components per grid
 * y.  loss_dev (optional device double): metrics.kl_div(norm q, norm V) of plca.py:245 with q = Hz W^T, without forming
 * q:  sum_nnz [t (log(t + eps) - log(x + eps)) - t] + norm sum_r colsum(W)[r] colsum(Hz)[r],  t = val norm and
 * x = norm (hz_n . w_c) in fp32 at each stored entry; the entries' terms come from the row gather's own pass (one double
 * partial per block), the column sums from double partials over row blocks, and one block sums them in a fixed order.
 * fp32 kernels; no atomics: every result is deterministic.  NMFB200_ERR_INVALID for another context kind, a null W or Hz,
 * or `out` and `loss_dev` both null; NMFB200_ERR_STATE before set_target.  Asynchronous. */
int nmfb200_plca_sparse_terms(nmfb200_ctx* ctx, const float* W, const float* Hz, float* out /* [dW | dHz] */, float norm,
                              double* loss_dev /* nullable */, void* stream);
/* Device bytes the context's workspace holds (the caller's buffers excluded); -1 for a null context or another kind. */
int64_t nmfb200_plca_sparse_device_bytes(const nmfb200_ctx* ctx);

/* ---- both models ------------------------------------------------------------------------- */

/* Every call below takes a context of either model and runs that model's kernels.  update_w, update_h, loss, raw_terms and
 * w_apply return NMFB200_ERR_STATE before the context's set_target*. */

/* Tell the engine the fp32 factors changed outside its own update calls (fit() entry, load_state_dict, a frozen factor,
 * a line search's trial factors): the tensor-core path keeps fp16 operand copies and refreshes only what it knows changed,
 * so both are rebuilt at the next call.  No device work. */
int nmfb200_sync_factors(nmfb200_ctx* ctx);

/* One W update, nmf.py:367-378:  W <- W * ((relu(Pn^T H)+eps) / den)^gamma  in place.
 * l1_reg / l2_reg as computed at nmf.py:348-349; gamma as nmf.py:341-346. */
int nmfb200_update_w(nmfb200_ctx* ctx, float* W, const float* H,
                     double beta, double gamma, double l1_reg, double l2_reg, void* stream);
/* One H update with the current (already updated) W, nmf.py:380-391. */
int nmfb200_update_h(nmfb200_ctx* ctx, const float* W, float* H,
                     double beta, double gamma, double l1_reg, double l2_reg, void* stream);
/* beta_div of the reconstruction against V (metrics.py:60-96) accumulated into the DEVICE double *loss_dev
 * (one element, overwritten).  Row / batch shards add: the sum over ranks is the global divergence. */
int nmfb200_loss(nmfb200_ctx* ctx, const float* W, const float* H, double beta, double* loss_dev, void* stream);

/* Raw terms of the multiplicative update of ONE factor (which = 0: W, 1: H), computed from the current W and H without
 * touching either: `out` receives the numerator relu-free (the factor's numel: the first backward pass of nmf.py:76-78 /
 * trainer.py:91-93), then colsum(other factor) (R, beta == 1: nmf.py:122-131) or the raw denominator (the factor's numel:
 * the second backward pass, nmf.py:82 / trainer.py:95-96); raw_terms_numel (-1 for a null context or a `which` other than
 * 0 and 1) is its length.  This is what torchnmf.trainer.BetaMu.step (trainer.py:36-121) and torchnmf.plca (plca.py:252-253:
 * the simultaneous W / H / Z updates from ONE V / (W Z H) ratio) are built from.
 *   NMFD / NMF2D / NMF3D: both backward passes through the conv1d / conv2d / conv3d reconstruction (nmf.py:776-779,
 *   :862-865, :938-942).  With W := W * Z this is one EM step's gradients of torchnmf.plca.SIPLCA / SIPLCA2 / SIPLCA3
 *   (plca.py:252-253 with the reconstructions :453-455, :534-537, :621-625).
 *   A sparse target (nmfb200_nmf_set_target_sparse) serves beta 1 and 2 with the same layout, from the same kernels as its
 *   update: the numerator at the non-zeros only, the beta-2 denominator F (other^T other); any other beta returns
 *   NMFB200_ERR_INVALID.  One set by nmfb200_nmf_set_target_sparse_any_beta also serves every other beta > 0 (2*rows*R
 *   floats: the numerator at the non-zeros, the V-free denominator equal bit for bit to a dense fp32 context's).
 * Sharded W update: every rank holds a shard of V and H (NMF: rows, the convolutive models: the batch axis) and a replica
 * of W.  raw_terms(which = 0) writes this shard's W terms; the caller sum-all-reduces the buffer and passes it to w_apply,
 * which runs the ratio stage nmf.py:78-92 on it, identically on every rank, and leaves the tensor-core state as update_w
 * does.  On one rank the pair is update_w bit for bit.  A sparse context gets its W terms too, in the layout and from the
 * kernels above. */
int64_t nmfb200_raw_terms_numel(const nmfb200_ctx* ctx, int which, double beta);
int nmfb200_raw_terms(nmfb200_ctx* ctx, const float* W, const float* H, int which, double beta, float* out, void* stream);

/* The gradient terms of one EM step of a PLCA / SIPLCA* fit on a partially observed target, from the current W and
 * Hz = H Z without touching either.  The mask M (nmfb200_set_mask) holds the observed cells O; the registered target is
 * Vn = V / sum_O V on O (its missing cells are never read); q = W Hz (NMF) or conv(Hz, W) (NMFD / NMF2D / NMF3D) the
 * model, q_O = sum_O q.  The EM step's ratio on the completed target is q_O M Vn / (q + eps) + (1 - M) q / (q + eps), so
 * the factor's gradient is q_O A + B with
 *   A = the backward pass of M Vn / (q + eps)        (the masked beta-1 numerator),
 *   B = the backward pass of (1 - M) q / (q + eps)   (the missing cells' fill term),
 * and `out` receives [A | B], each the factor's numel (which = 0: W, 1: Hz), raw-summed as nmfb200_raw_terms' slabs.
 * qobs_dev (optional device double): q_O, from one partial per block of the same pass summed in a fixed order.  One
 * contraction pass over V and M per call, as nmfb200_raw_terms at beta 1.  fp32 CUDA-core kernels, fp32 V; NMFD / NMF2D /
 * NMF3D up to rank 256.  NMFB200_ERR_STATE before set_target or without a mask; NMFB200_ERR_INVALID for a weight, a
 * sparse, observed-cell or batched context, a non-fp32 target, or an NMFD rank above 256.  Asynchronous. */
int nmfb200_plca_masked_terms(nmfb200_ctx* ctx, const float* W, const float* Hz, int which, float* out, double* qobs_dev,
                              void* stream);
int nmfb200_w_apply(nmfb200_ctx* ctx, float* W, const float* reduced, double beta, double gamma, double l1_reg,
                    double l2_reg, void* stream);

/* Fit only the observed cells of a dense target.  M: a DEVICE array of uint8 in V's shape, contiguous (NMF: N x C whatever
 * V's ldv; the convolutive models: V's layout), non-zero = observed; borrowed like V.  Valid after nmfb200_nmf_set_target /
 * nmfb200_nmfd_set_target (NMFB200_ERR_STATE before), NMFB200_ERR_INVALID on a sparse context.  A null M, or any later
 * set_target*, clears the mask (contexts are reused between fits).  While a mask is set the loss is
 * beta_div(WH[M], V[M]) -- the missing cells dropped, not zeroed -- and every update is nmf.py:78-92 applied to the two
 * backward passes of that loss: num = (M * v x^(beta-2)) G, den = (M * x^(beta-1)) G, so at beta 1 den = M G instead of the
 * column sums of G.  The kernels select, they never multiply by the mask: V is not read at a missing cell, so a NaN, Inf or
 * negative value there gives the bits a zero gives.  update_w, update_h, nmf_iterate, loss, nmf_loss_prefetch_w (= loss),
 * raw_terms (raw_terms_numel: 2 x the factor's numel at every beta), w_apply, contract_only and target_minmax (observed
 * cells only) follow it; they run on the fp32 CUDA-core kernels (precision_for_beta reports NMFB200_PREC_F32,
 * nmf_peer_supported 0) and leave the tensor-core operand copies marked stale.  Asynchronous. */
int nmfb200_set_mask(nmfb200_ctx* ctx, const uint8_t* M, void* stream);

/* Fit a dense target with per-cell weights.  Wt: a DEVICE array of fp32 in V's shape, contiguous (NMF: N x C whatever V's
 * ldv; the convolutive models: V's layout), borrowed like V; every weight finite and >= 0 (not checked here).  Same contract
 * as nmfb200_set_mask: valid after a dense set_target (NMFB200_ERR_STATE before), NMFB200_ERR_INVALID on a sparse or
 * observed-cell context; a null Wt, or any later set_target*, clears it; set_mask and set_weight replace each other.  While
 * a weight is set the loss is sum_{w > 0} w d_beta(v | x), and every update is nmf.py:78-92 applied to the two backward
 * passes of that loss: num = (w v x^(beta-2)) G, den = (w x^(beta-1)) G (beta 1: den = Wt G).  The kernels multiply where
 * the mask kernels select: a cell of weight 0 is dropped, V is not read there (NaN, Inf or a negative value there gives
 * the bits a zero gives), and a weight of exactly 1 gives the bits of a mask.  Every call that follows a mask follows the
 * weight: update_w, update_h, nmf_iterate, loss, nmf_loss_prefetch_w (= loss), raw_terms (2 x the factor's numel at every
 * beta), w_apply, contract_only and target_minmax (the cells with w != 0), on the fp32 CUDA-core kernels
 * (precision_for_beta reports NMFB200_PREC_F32, nmf_peer_supported 0).  Asynchronous. */
int nmfb200_set_weight(nmfb200_ctx* ctx, const float* Wt, void* stream);

/* Hold chosen components of W at their values (semi-supervised fits: a dictionary learned beforehand stays fixed while the
 * other components learn the rest of the target).  fixed: a DEVICE array of R uint8, non-zero for a fixed component k
 * (W[:, k] for NMF, W[:, k, ...] for NMFD / NMF2D / NMF3D), borrowed like a mask.  Valid on a single NMF or NMFD context
 * after any set_target* (NMFB200_ERR_STATE before); NMFB200_ERR_INVALID on batched and sparse-PLCA contexts.  A null fixed,
 * or any later set_target*, clears it.  While it is set, every call that writes W -- update_w, nmf_iterate, w_apply,
 * nmf_cd_update / _iterate and nmf_observed_cd_update / _iterate, on every kernel family -- leaves the fixed components
 * unstored: the free ones take exactly the update they take without it (the reconstruction formed from all R components,
 * the penalties on the free ones only), and a fixed component still enters the tensor-core operand scale, column sums and
 * loss as it is.  The coordinate-descent sweeps skip each fixed k: no step, and later components see its unchanged value.
 * H updates are unaffected, and nmf_peer_supported reports 0 while it is set.  Queues nothing. */
int nmfb200_set_fixed_w(nmfb200_ctx* ctx, const uint8_t* fixed, void* stream);

/* Automatic relevance determination with the l1 prior (Tan and Fevotte, TPAMI 2013): component k has a relevance lambda_k,
 * and every W and H update adds pen_k = phi / lambda_k to the denominator of component k's elements, with the fp32 add of the
 * scalar l1_reg (pass l1_reg = l2_reg = 0 for the ARD objective).  Registration: W and H are the factors the fit starts
 * from (read here, not kept); b, c and phi (finite, > 0) the prior's scale, c = n_W + n_H + a + 1 and the dispersion.  It
 * sets lambda_k = (sum W[:, k] + sum H[:, k] + b) / c, pen_k = phi / lambda_k and the change to 0 (the sums over every entry
 * of component k, W[:, k, ...] and H[:, k, ...] for NMFD / NMF2D / NMF3D; fixed-order fp32 column sums, the rest in double,
 * lambda and pen stored as fp32).  The context owns lambda, pen and the change.  W and H both null clear the registration,
 * and so does any later set_target*.  Valid on a single NMF or NMFD context after any set_target* (NMFB200_ERR_STATE
 * before); NMFB200_ERR_INVALID on batched and sparse-PLCA contexts and while nmfb200_set_fixed_w holds components (and
 * set_fixed_w refuses the same way while ARD is registered).  While it is registered: update_w, update_h and nmf_iterate
 * add pen on every kernel family; nmf_iterate runs, each iteration, the W update, the H update, then nmfb200_ard_update;
 * loss_prefetch_w stays valid (the lambda update moves no factor); nmf_peer_supported reports 0, and nmf_update_w_peer,
 * w_apply, nmf_cd_* and nmf_observed_cd_* return NMFB200_ERR_INVALID.  Asynchronous. */
int nmfb200_set_ard(nmfb200_ctx* ctx, const float* W, const float* H, double b, double c, double phi, void* stream);

/* The lambda update from the current W and H: lambda_k as at registration, pen_k = phi / lambda_k, and the change
 * max_k |lambda_k - previous lambda_k| / previous lambda_k.  Deterministic: no float atomics.  NMFB200_ERR_STATE without
 * a registration.  Asynchronous. */
int nmfb200_ard_update(nmfb200_ctx* ctx, const float* W, const float* H, void* stream);

/* Copies lambda (R floats), pen (R floats) and the change (one float) to the non-null pointers among lambda / pen /
 * change, host or device memory, then synchronises `stream`.  NMFB200_ERR_STATE without a registration. */
int nmfb200_ard_read(nmfb200_ctx* ctx, float* lambda, float* pen, float* change, void* stream);

/* ---- tile plans of the fp32 CUDA-core kernels (host only: no device work, no allocation) -------- */

/* What a context of these sizes runs on the fp32 kernels, from the library's own planners.  `out` receives
 * NMFB200_NMF_PLAN_LEN values (n must be at least that):
 *   [0] chunks of the W update's contraction over the N rows    [1] chunks of the H update's over the C columns
 *   [2] 64-wide tiles per chunk, W update                       [3] the same, H update (the last chunks may be short or empty)
 *   [4] register blocks RB of the contraction (rank <= 16 RB up to 256; above, 16 RB = 256 components per rank block,
 *       ceil(R / 256) blocks on grid z)   [5] chunks of the loss pass   [6] its tiles per chunk
 *   [7] blocks of the column sum over N rows (the W update's KL denominator)   [8] over C rows (the H update's) */
#define NMFB200_NMF_PLAN_LEN 9
int nmfb200_nmf_plan(int64_t N, int64_t C, int64_t R, int64_t* out, int n);
/* The same for the sparse-target kernels of an (N, C) rank-R context, NMFB200_SPARSE_PLAN_LEN values:
 *   [0] rank floats per lane of the warp-per-row kernels (1, 2, 4, 8)   [1] Gram passes of 4096 (a, b) pairs
 *   [2] Gram rows per block over the N rows of H (a multiple of 32)   [3] its blocks (at most 128, the last may be short)
 *   [4], [5] the same over the C rows of W   [6] blocks (8 rows each) over N: the H update's gathers and the loss's partials
 *   [7] over C: the W update's
 * An observed-cell context (nmfb200_nmf_set_target_observed) runs its terms and loss gathers on [0], [6] and [7] and
 * launches no Gram kernel. */
#define NMFB200_SPARSE_PLAN_LEN 8
int nmfb200_nmf_sparse_plan(int64_t N, int64_t C, int64_t R, int64_t* out, int n);
/* The same for an NMFD / NMF2D / NMF3D context (arguments as nmfb200_nmfnd_create), NMFB200_NMFD_PLAN_LEN values:
 *   [0] recon row tile MT (channels)   [1..3] recon grid x, y, z of one launch
 *   [4] dgrad row tile MT (components)   [5] dgrad splits of C   [6..8] dgrad grid x, y, z of one launch
 *   (z = batch elements per launch, at most 65535: a larger batch takes ceil(B / z) launches)
 *   [9..15] wgrad plan mt, tp, nr, no, ntt, nrg, nog   [16] wgrad splits of the lines
 *   [17], [18] 1 if the W / H ratio stage takes the four-elements-per-thread kernel, else 0 */
#define NMFB200_NMFD_PLAN_LEN 19
int nmfb200_nmfd_plan(int64_t B, int64_t C, int ndim, const int64_t* vdims, int64_t R, const int64_t* kdims,
                      int64_t* out, int n);
/* What the tensor-core (beta 1) kernels of an NMFD / NMF2D / NMF3D context (arguments as nmfb200_nmfnd_create) launch, from
 * the planner those launches use; NMFB200_ERR_INVALID, naming the limit, for a shape that create rejects with precision f16
 * (and NMFD runs on the fp32 kernels with precision auto).  NMFB200_NMFND_TC_PLAN_LEN values:
 *   [0..2] prep_w grid   [3..5] prep_h grid   [6..8] recon grid of one launch   [9..11] wgrad grid
 *   [12..14] dgrad grid of one launch   [15] target lines (b, x1, x2) per recon launch (grid z)   [16] recon launches
 *   (line slices)   [17] dgrad launches per slice (blocks of 128 components)   [18] recon-loss partials over all lines
 *   [19] wgrad splits   [20] wgrad k-blocks per split   [21] dgrad splits   [22] dgrad k-blocks per split
 *   [23] activation lines (b, j1, j2) per dgrad launch (grid z)   [24] dgrad launches (line slices)
 *   [25] Tp (T rounded up to 64)   [26] H copy left margin   [27] H copy row pitch   [28] ratio tile row pitch
 *   [29] C rounded up to 128   [30] 2048-element chunks per H row (prep_h)
 * Whatever the number of axes, a shape whose outer sizes are all 1 plans as its one-axis NMFD shape. */
#define NMFB200_NMFND_TC_PLAN_LEN 31
int nmfb200_nmfnd_tc_plan(int64_t B, int64_t C, int ndim, const int64_t* vdims, int64_t R, const int64_t* kdims,
                          int64_t* out, int n);
/* What the tensor-core contraction of a dense (N, C) rank-R NMF context (nmfb200_nmf_create) launches on a device with
 * num_sms SMs, from the planner and the shared-memory layout those launches use; precision f16 or f16_split (auto plans as
 * f16).  The kernel is persistent: grid CTAs, CTA b walks the work items b, b + grid, b + 2 grid, ... (item = chunk x
 * row_blocks + row block).  NMFB200_ERR_INVALID for f32, sizes below 1, num_sms below 1, and shapes create refuses at f16.
 * NMFB200_NMF_TC_PLAN_LEN values:
 *   [0] TN, columns of V per tile   [1] NS, stages of the tile ring   [2] NF, F blocks (1 or 2) the producer loads ahead
 *   [3..8] the W update (rows C, contracted over N): row blocks of 128, tiles, chunks, tiles per chunk (the last chunk
 *   may be short), items, grid   [9..14] the same for the H update and the loss (rows N, contracted over C) */
#define NMFB200_NMF_TC_PLAN_LEN 15
int nmfb200_nmf_tc_plan(int64_t N, int64_t C, int64_t R, int precision, int num_sms, int64_t* out, int n);

/* ---- sparseness-constrained NMF (Hoyer 2004) --------------------------------------------- */

/* Replaces torchnmf.nmf._proj_func (nmf.py:21-49) and the Python loops that call it once per component
 * (sparse_fit nmf.py:462-465, :472-475, :519-522, :565-568; trainer.SparsityProj.step trainer.py:176-181): every slice
 * x[:, j, :] of the fp32 device tensor x viewed as (outer, D, inner) is replaced IN PLACE by the closest non-negative
 * vector with L1 norm k1[j] and squared L2 norm k2[j] (k1, k2: D device floats).  The reference's data-dependent loop
 * (one host synchronisation per round and slice) runs on the device, one block per slice, one launch for all D slices.
 * zeroed_ws: D * outer * inner bytes of device scratch, any contents (cleared in the first round).  Context-free: runs on
 * CUDA device `device`, the caller's current device is restored.
 * Degenerate slices, as the reference's arithmetic has them: where the surviving support is uniform after fp32 rounding
 * (a constant slice, survivors that all tie, or one element whose shifted value x + (k1 - x) rounds exactly to k1)
 * w.w = 0 and the quadratic gives 0 / 0, so the slice becomes NaN, as in the reference; a one-element slice whose shift
 * does not round exactly keeps w != 0 and a finite result.  Where a round zeroes every coordinate the reference divides by zero (ZeroDivisionError); the kernel stops
 * and leaves the slice at zero.  fp32 rounding decides which of the two a near-uniform slice meets: float64 and fp32 can
 * differ there. */
int nmfb200_hoyer_project(int device, float* x, int64_t outer, int64_t D, int64_t inner, const float* k1, const float* k2,
                          void* zeroed_ws, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NMF_B200_H_ */
