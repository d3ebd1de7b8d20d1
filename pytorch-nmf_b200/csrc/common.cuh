// Shared declarations for the libnmf_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <type_traits>

namespace nmfb200 {

// torchnmf/constants.py:3 -- float32 machine epsilon, 2^-23
constexpr float kEps = 1.1920928955078125e-07f;

// Element type of the dense target V (include/nmf_b200.h: NMFB200_DTYPE_*).  Every kernel that reads V takes it as a
// template parameter TV and converts each element with to_f32 where it loads it.  fp16 and bf16 values are exact in fp32,
// so everything after the load computes what it computes on an fp32 copy of the same values.
enum VDtype : int { kVF32 = 0, kVF16 = 1, kVBF16 = 2 };
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
// bf16 is the upper half of an fp32 word: the same bits as __bfloat162float, written as the integer shift because that form
// leaves the fp32 CUDA-core contraction's register allocation as it is for fp32 (no extra spill in its beta != 0, 1, 2 kernels)
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __uint_as_float((unsigned)__bfloat16_as_ushort(v) << 16); }
static inline int vdtype_size(int dtype) { return dtype == kVF32 ? 4 : 2; }
// Host dispatch: f(p) with p = V as `const float*`, `const __half*` or `const __nv_bfloat16*` per `dtype` (validated by the
// caller: capi.cu's set_target); vtype_t<decltype(p)> is the element type.
template <class P>
using vtype_t = std::remove_cv_t<std::remove_pointer_t<P>>;
template <class F>
int with_vtype(const void* V, int dtype, F&& f) {
  if (dtype == kVF16) return f(static_cast<const __half*>(V));
  if (dtype == kVBF16) return f(static_cast<const __nv_bfloat16*>(V));
  return f(static_cast<const float*>(V));
}

// Per-cell selector of a dense fit (nmfb200_set_mask / nmfb200_set_weight): none, a uint8 mask (the kernels select the
// observed cells) or fp32 weights (the kernels multiply each cell's terms by its weight, and drop the cells of weight 0).
// Kernels take the selector's element type as a template parameter SEL: NoSel, uint8_t or float.
enum SelKind : int { kSelNone = 0, kSelMask = 1, kSelWeight = 2 };
struct NoSel {};
struct CellSel {
  const void* p = nullptr;
  int kind = kSelNone;
  explicit operator bool() const { return p != nullptr; }
};
template <class P>
using sel_t = std::remove_cv_t<std::remove_pointer_t<P>>;
template <class SEL>
constexpr bool kWeighted = std::is_same<SEL, float>::value;
// whether cell i takes part in the fit: always without a selector, else where M is non-zero
template <class SEL>
__device__ __forceinline__ bool sel_set(const SEL* M, int64_t i) {
  if constexpr (std::is_same<SEL, NoSel>::value) return true;
  else return M[i] != 0;
}
// Host dispatch: f(p) with p = the selector as `const NoSel*` (null), `const uint8_t*` or `const float*`
template <class F>
int with_sel(CellSel s, F&& f) {
  if (s.p && s.kind == kSelWeight) return f(static_cast<const float*>(s.p));
  if (s.p) return f(static_cast<const uint8_t*>(s.p));
  return f(static_cast<const NoSel*>(nullptr));
}

// One problem of a ragged batch (nmfb200_nmf_batched_create_ragged): N_b <= N rows over the batch's C columns, stored in
// the padded (B, N, ...) layouts of V and H.  It runs the plan of a single problem of N_b rows: its own chunk counts, loss
// chunks and column-sum blocks, and its partials laid out as that problem's, at its own offsets in the shared buffers.  Its
// blocks of each launch below start at x0[launch] on grid x and run up to the next problem's (x0 ascends with b).
// A ragged batch of NMFD / NMF2D / NMF3D problems (nmfb200_nmfnd_batched_create_ragged) uses the same table: `rows` is then
// L_p, the problem's length along the sliding axis of the padded (P, B, C, *X) target, and `lin` = L_p - T + 1 its
// activation positions there.  Its launches put the problems' lines on grid z (no x0, no search): each sizes grid x / y for
// the largest problem, and a problem's blocks past its own grid x (gx) or dgrad splits (nch[1]) exit at once.  Its ratio
// tiles Pn / Pp are the single problem's (B, C, *X[:-1], L_p) at `pn`, its wgrad / dgrad split slabs ([split][C, R, K] /
// [split][B, R, *J[:-1], lin]) at `part`, its loss partials at `loss_part` and its column-sum partials of H at `cs_part`.
enum RaggedLaunch : int { kRagW = 0, kRagH = 1, kRagLoss = 2, kRagColsum = 3 };
struct RaggedProblem {
  int64_t rows;           // N_b (NMFD: L_p)
  int64_t x0[4];          // first block on grid x of the W and H contractions, the loss and the column sums of H
  int64_t part;           // floats before its partial slabs ([chunk][rows][R], rows = C for W and N_b for H)
  int64_t loss_part;      // doubles before its loss partials ([chunk][row block])
  int64_t cs_part;        // floats before its column-sum partials of H ([block][R])
  int64_t loss_n;         // its loss partials
  int nch[2];             // contraction chunks of its W / H update (NMFD: wgrad / dgrad splits)
  int loss_chunks;
  int cs_blocks;          // column-sum blocks over its rows
  int64_t pn;             // NMFD: floats before its ratio tiles
  int lin;                // NMFD: L_p - T + 1
  int gx[2];              // NMFD: grid x of its recon (FWD) and dgrad slides
};
// the problem of a ragged batch's n whose blocks of `launch` hold grid-x block bx: the last one with x0[launch] <= bx
__device__ __forceinline__ int64_t ragged_problem(const RaggedProblem* t, int64_t n, int launch, int64_t bx) {
  int64_t lo = 0, hi = n - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (t[mid].x0[launch] <= bx) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// A batch of independent NMF problems of one shape (nmfb200_nmf_batched_create).  The kernels that take it run every problem
// in one launch, with the batch folded into grid x: problem b owns the blocks [b nbx, (b + 1) nbx) of the nbx blocks one
// problem launches, and does in them exactly what a launch for that problem alone does.  Offsets between problems are in
// elements of the pointer they apply to, int64.  The default is one problem (every single-problem call).
// A ragged batch (rag set: n problems' plans in device memory) keeps v, f and g -- V and the factors stay padded -- and takes
// each problem's rows, chunks, partial offsets and first block from rag[b] instead; the launch's grid x is rag_gx, its
// grid y 1 (the chunks ride on grid x too).
struct Batch {
  int64_t n = 1;                      // problems
  int64_t v = 0;                      // target elements between problems (0: one target shared by every problem)
  int64_t f = 0, g = 0;               // floats between problems' F / G factors of a contraction or loss
  int64_t p = 0;                      // floats between problems' partial slabs (within one chunk)
  const uint8_t* active = nullptr;    // n flags, 0 = skipped: the problem's blocks exit at once (null: every problem runs)
  // KL loss only (batched PLCA): n floats, problem b's target and reconstruction are multiplied by scale[b] before the loss
  // term (null: none)
  const float* scale = nullptr;
  const RaggedProblem* rag = nullptr; // ragged batch: n per-problem plans (null: every problem has the launch's shape)
  int rag_launch = 0;                 // RaggedLaunch of this launch
  int64_t rag_gx = 0;                 // its grid x: the sum of the problems' blocks
};
__device__ __forceinline__ bool batch_skips(const uint8_t* active, int64_t b) { return active && !active[b]; }

// beta-divergence branch of nmf.py:61-74 / metrics.py:60-96
enum BetaMode : int { kKL = 0, kEU = 1, kIS = 2, kGeneric = 3 };
// The term mode of a masked PLCA fit (nmfb200_plca_masked_terms), beside BetaMode (and simt_nmf.cu's kVFree = 4): with the
// uint8 mask, Pn = v / (s + eps) at an observed cell and 0 elsewhere, Pp = s / (s + eps) at a missing cell and 0 elsewhere,
// and the pass sums s over the observed cells it covers into one double partial per block.  fp32 V, one problem.
constexpr int kPlcaFill = 5;
inline BetaMode beta_mode(double beta) {
  if (beta == 1.0) return kKL;
  if (beta == 2.0) return kEU;
  if (beta == 0.0) return kIS;
  return kGeneric;
}

// one cell's term of metrics.beta_div (metrics.py:60-96): v the target, s the reconstruction, in fp32; shared by the dense
// loss kernels (simt_nmf.cu) and the observed-cell gathers (sparse_nmf.cu)
template <int MODE>
__device__ __forceinline__ float loss_term(float v, float s, float beta) {
  if (MODE == kKL) {               // metrics.py:22
    return v * (logf(v + kEps) - logf(s + kEps)) - v + s;
  } else if (MODE == kEU) {        // metrics.py:39
    float d = s - v;
    return 0.5f * d * d;
  } else if (MODE == kIS) {        // metrics.py:56-57
    float te = v + kEps, xe = s + kEps;
    return te / xe - logf(te) + logf(xe) - 1.0f;
  } else {                         // metrics.py:84-96
    float x = s + kEps;
    float t = beta < 0.f ? v + kEps : v;
    float bm = beta - 1.0f;
    return (powf(t, beta) + bm * powf(x, beta) - beta * t * powf(x, bm)) / (beta * bm);
  }
}

// w * loss_term, with w folded into the product the caller's accumulation fuses with at beta 2, so that w = 1 gives the
// bits of the unweighted term's accumulation and w = 2^k exactly 2^k times them
template <int MODE>
__device__ __forceinline__ float loss_term_w(float v, float s, float beta, float w) {
  if (MODE == kEU) {
    float d = s - v;
    return (0.5f * w * d) * d;
  }
  return w * loss_term<MODE>(v, s, beta);
}

void set_error(const std::string& msg);
void count_launch();

#define NMF_CUDA_CHECK(expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      nmfb200::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));             \
      return 2;                                                                           \
    }                                                                                     \
  } while (0)

#define NMF_LAUNCH_CHECK()                                                                \
  do {                                                                                    \
    nmfb200::count_launch();                                                              \
    cudaError_t _e = cudaGetLastError();                                                  \
    if (_e != cudaSuccess) {                                                              \
      nmfb200::set_error(std::string("kernel launch: ") + cudaGetErrorString(_e));        \
      return 2;                                                                           \
    }                                                                                     \
  } while (0)

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int64_t round_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// CUDA's grid limits: x up to 2^31 - 1 blocks, y and z up to 65535
constexpr int64_t kMaxGridX = 0x7fffffff;
constexpr int64_t kMaxGridYZ = 65535;
// a launch's grid as planned on the host, before it is narrowed to dim3
struct Grid3 { int64_t x, y, z; };
static inline bool grid_fits(const Grid3& g) {
  return g.x >= 1 && g.x <= kMaxGridX && g.y >= 1 && g.y <= kMaxGridYZ && g.z >= 1 && g.z <= kMaxGridYZ;
}

// ------------------------------------------------------------------------------------------
// Launch wrappers implemented in the .cu files (all asynchronous on `st`, return 0 / error code)
// ------------------------------------------------------------------------------------------

// simt_nmf.cu ------------------------------------------------------------------------------
// Partial contractions of one factor update on CUDA cores, fp32:
//   S = F G^T (Mr x Nc),  (Pn, Pp) = phi_beta(Vm, S)          [nmf.py:61-74]
//   num[ch][m][r] = sum_{c in chunk ch} Pn[m,c] G[c,r]          [nmf.py:77]
//   den[ch][m][r] = sum_{c in chunk ch} Pp[m,c] G[c,r]          [nmf.py:82, beta != 1 only]
// Vm[m,c] = V[m*ldv + c] (trans = 0) or V[c*ldv + m] (trans = 1), elements of type `vdtype` (VDtype).  Any rank R >= 1.
// M (optional selector, read like V with pitch ldm): a fit on the observed cells only -- Pn = Pp = 0 where M is 0, V is not
// read there, and den is always formed (beta 1: Pp = M).  A weight selector multiplies Pn and Pp by the cell's weight
// (beta 1: Pp = the weight).  An empty M runs the unmasked kernels.
// bt: bt.n problems in one launch (no selector then), problem b reading V + b bt.v, F + b bt.f, G + b bt.g and writing its
// slabs at num / den + b bt.p.
int simt_nmf_contract(const void* V, int vdtype, int64_t ldv, int trans, const float* F, const float* G,
                      int64_t Mr, int64_t Nc, int R, double beta, int nchunks,
                      float* num, float* den, int64_t ldp, int64_t chunk_stride, CellSel M, int64_t ldm,
                      cudaStream_t st, const Batch& bt = Batch{});
// beta_div(F G^T, Vm) accumulated into block partials then *loss_dev (double); over the cells where M (optional, pitch
// ldm, not transposed) is non-zero, each term times the cell's weight for a weight selector.  bt: loss_dev[b] for problem
// b, from its own run of partials summed in the single problem's order; a skipped problem's slot is left as it is.
int simt_nmf_loss(const void* V, int vdtype, int64_t ldv, const float* F, const float* G, int64_t Mr, int64_t Nc,
                  int R, double beta, double* block_partials, int max_blocks, double* loss_dev, CellSel M,
                  int64_t ldm, cudaStream_t st, const Batch& bt = Batch{});
int simt_nmf_max_blocks(int64_t Mr, int64_t Nc);
// The terms of one factor of a masked PLCA fit on simt_nmf_contract's plan at beta 1 (kPlcaFill), fp32 V, uint8 mask M:
//   num[ch][m][r] = sum_{c in chunk ch} M Vm[m,c] / (S[m,c] + eps) G[c,r]
//   den[ch][m][r] = sum_{c in chunk ch} (1 - M) S[m,c] / (S[m,c] + eps) G[c,r]
// and, when qobs_part is not null, qobs_part[ch * ceil(Mr / 64) + row block] = the sum of S over the observed cells of that
// block's tiles (rank-blocked plans: output block 0 only), simt_plca_fill_blocks of them.
int simt_plca_fill_contract(const float* V, int64_t ldv, int trans, const float* F, const float* G, int64_t Mr, int64_t Nc,
                            int R, int nchunks, float* num, float* den, int64_t ldp, int64_t chunk_stride, const uint8_t* M,
                            int64_t ldm, double* qobs_part, cudaStream_t st);
int64_t simt_plca_fill_blocks(int64_t Mr, int nchunks);
// The V-free pieces of a sparse target's update and loss at beta != 1, 2 (nmf.py:621-636):
//   den[ch][m][r] = sum_{c in chunk ch} (S[m,c] + eps)^(beta-1) G[c,r]: simt_nmf_contract's denominator at this beta, bit for
//   bit (same grid, chunks and arithmetic), without reading V; R <= 256.
int simt_nmf_contract_den(const float* F, const float* G, int64_t Mr, int64_t Nc, int R, double beta, int nchunks,
                          float* den, int64_t ldp, int64_t chunk_stride, cudaStream_t st);
//   block_partials[*nblocks] of sum over every cell of (S + eps)^beta (fp32 terms, double block sums), on simt_nmf_loss's plan.
int simt_nmf_pow_sum(const float* F, const float* G, int64_t Mr, int64_t Nc, int R, double beta, double* block_partials,
                     int max_blocks, int* nblocks, cudaStream_t st);
// The numerator alone of simt_nmf_contract at beta 2 (kNumOnly), no selector, R <= 256:
//   num[ch][m][r] = sum_{c in chunk ch} Vm[m,c] G[c,r]     (row pitch R)
// bit for bit simt_nmf_contract's num partials at beta 2 (same grid, chunks, staging and loop order), without S = F G^T.
// bt: as simt_nmf_contract's (bt.f unused), problem b reading V + b bt.v, G + b bt.g and writing num + b bt.p.
int simt_nmf_contract_num(const void* V, int vdtype, int64_t ldv, int trans, const float* G, int64_t Mr, int64_t Nc, int R,
                          int nchunks, float* num, int64_t chunk_stride, cudaStream_t st, const Batch& bt = Batch{});
// Output blocks of 256 components of simt_nmf_contract (grid z): 1 up to rank 256, each block recomputes S over all ranks.
int simt_rank_blocks(int R);
// The tile plan of simt_nmf_contract (Mr rows, Nc contracted columns, `nchunks` chunks) and of simt_nmf_loss: the register
// blocks RB of 16 components, the 64-column tiles per chunk (the last chunks may be short or empty) and the loss's chunks.
struct SimtNmfPlan { int rb; int64_t tiles_per_chunk; int loss_chunks; int64_t loss_tiles_per_chunk; };
void simt_nmf_plan(int64_t Mr, int64_t Nc, int R, int nchunks, SimtNmfPlan* p);

// Gram matrix out = F^T F (R x R) of a (rows x R) fp32 factor, R <= 256: one partial per block (sparse_gram_part_floats(R)
// floats of `part`), then a sum over the blocks in fixed order (sparse_nmf.cu; serves the sparse beta-2 path and cd.cu).
// bt: bt.n problems in the same two launches, problem b's F at F + b bt.f and its Gram at out + b bt.p, each on the single
// problem's sparse_gram_plan(rows) blocks and summation order; its nb R^2 partials are the b-th run of `part`.
int sparse_gram(const float* F, int64_t rows, int R, float* part, float* out, cudaStream_t st, const Batch& bt = Batch{});
int64_t sparse_gram_part_floats(int R);

// cd.cu ------------------------------------------------------------------------------------
// One HALS sweep of a (rows x R) factor X in place, R <= 256 (nmfb200_nmf_cd_update): with A = the sum over `nchunks` slabs
// (chunk_stride apart, row pitch R) of the numerator partials, in raw_sum's order, and B (R x R), for k = 0 .. R-1 in order
//   X[c,k] <- max(0, X[c,k] + (A[c,k] - sum_j X[c,j] B[j,k] - l1 - l2 X[c,k]) / (B[k,k] + l2))
// on every row c, columns with B[k,k] + l2 == 0 left as they are.  bt: bt.n problems in one launch, problem b's X at
// X + b bt.f, its A partials at A + b bt.p within each slab and its B at B + b bt.g, each summed in the single problem's
// order; problems whose bt.active flag is 0 are left untouched.  fixed (R bytes, one problem only; null: none): the sweep
// skips every column k with fixed[k] != 0, which keeps its value, and later columns see that value.
int cd_sweep(float* X, int64_t rows, int R, const float* A, int nchunks, int64_t chunk_stride, const float* B, float l1,
             float l2, cudaStream_t st, const Batch& bt = Batch{}, const uint8_t* fixed = nullptr);
// blocks of one problem's sweep over `rows` rows (grid x: this times the problems of a batch)
int64_t cd_sweep_blocks(int64_t rows);

// observed_cd.cu ---------------------------------------------------------------------------
// One coordinate-descent update of a (nseg x R) factor X in place on the observed cells, R <= 256
// (nmfb200_nmf_observed_cd_update): ptr / idx / val (and the entries' weights wt, null: unweighted) the compressed form whose
// segments are X's rows, F the other factor.  rbuf: observed_cd_workspace_floats(R, nnz) floats (none for R <= 32).
// fixed (R bytes; null: none): the sweep skips every component k with fixed[k] != 0 -- no step, no residual update.
int observed_cd(const int64_t* ptr, const int64_t* idx, const float* val, const float* wt, float* X, const float* F, int R,
                int64_t nseg, float* rbuf, float l1, float l2, cudaStream_t st, const uint8_t* fixed = nullptr);
int64_t observed_cd_workspace_floats(int R, int64_t nnz);

// update.cu --------------------------------------------------------------------------------
// nmf.py:78-92 on a flattened parameter of `numel` elements whose rank index is
// r = (idx / inner) % R.   num/den are sums over `nchunks` partial slabs (stride chunk_stride,
// row pitch ldp for a (rows x R*inner) view: element idx -> (idx / rowlen) * ldp + idx % rowlen).
struct ApplyArgs {
  float* param; int64_t numel; int R; int64_t inner; int64_t rowlen;
  const float* num; const float* den; int nchunks; int64_t chunk_stride; int64_t ldp;
  const float* kl_den;     // [R] when beta == 1 (den == nullptr)
  const float* out_scale;  // device scalar multiplying num/den partials (nullptr = 1)
  float gamma, l1, l2;
  unsigned int* absmax_bits;  // optional: atomicMax of the updated values (non-negative floats)
  const float* kappa;         // optional (with kappa_vec): the partials hold sum (P - kappa) G; num += *kappa * kappa_vec[r]
  const float* kappa_vec;     // [R]
  // a batch of problems (Batch): every prob_numel consecutive elements are one problem's, which takes its kl_den at
  // kl_den + b R; a problem whose active flag is 0 is left untouched (0: one problem)
  int64_t prob_numel = 0;
  const uint8_t* active = nullptr;
  // a ragged batch (Batch::rag, with prob_numel): problem b's partials are its own nch[rag_launch] slabs at rag[b].part, of
  // its rows (kRagH: rag[b].rows, kRagW: all prob_numel / rowlen) x ldp; nchunks and chunk_stride are not read.  The rows of
  // H past rag[b].rows are padding: left untouched.
  const RaggedProblem* rag = nullptr;
  int rag_launch = 0;
  // a ragged NMFD batch's H (kRagH): the padded length of the sliding axis, the last of H's (R, *J) inner axes.  Element
  // (line, j) of problem b is real for j < rag[b].lin, its partials at rag[b].part + line rag[b].lin + j in slabs of the
  // problem's compact size; the others are padding, left untouched.  0: the layout above
  int64_t line = 0;
};
// fixed (R bytes, one problem only; null: none): the elements of every component r with fixed[r] != 0 are not stored
// (they keep their value, which is what an absmax_bits update takes for them).  pen (R floats, one problem only, exclusive
// with fixed; null: none): the ARD penalties, pen[r] added to the denominator of every element of component r after a.l1.
int apply_update(const ApplyArgs& a, cudaStream_t st, const uint8_t* fixed = nullptr, const float* pen = nullptr);
// whether apply_update takes its four-elements-per-thread kernel for this shape (16-byte aligned buffers provided)
bool apply_update_vec4_shape(const ApplyArgs& a);
// num_out[i] (and den_out[i] when a.den) = what the ratio stage would read for element i: summed partials + centring term
int raw_sum(const ApplyArgs& a, float* num_out, float* den_out, cudaStream_t st);
// sums[r] = sum over all other dims of x viewed as (outer, R, inner); deterministic two-stage.  nprob > 1: sums[b R + r] for
// nprob consecutive (outer, R, inner) problems, each summed in the single problem's order, skipping those whose `active`
// flag is 0; scratch_floats then covers nprob x colsum_scratch_floats.  rag (inner 1; a ragged batch's table): problem b
// sums its rag[b].rows rows of its (outer, R) block on its own rag[b].cs_blocks blocks, partials at rag[b].cs_part; rag_gx
// is their sum.  rag with rag_line (a ragged NMFD batch's H, inner > 1, its last axis rag_line long): problem b sums the
// first rag[b].lin positions of every line, in the order and blocking of a single problem's inner = inner / rag_line
// rag[b].lin (rows blocking when that is 1), partials at rag[b].cs_part.
int factor_colsum(const float* x, int64_t outer, int R, int64_t inner, float* scratch, int64_t scratch_floats,
                  float* sums, cudaStream_t st, int64_t nprob = 1, const uint8_t* active = nullptr,
                  const RaggedProblem* rag = nullptr, int64_t rag_gx = 0, int64_t rag_line = 0);
int64_t colsum_scratch_floats(int64_t outer, int R, int64_t inner);
// min / max of a strided matrix of `vdtype` elements (fit()'s validation), results in mm[0..1]; with M (optional, contiguous
// rows x cols selector) over the cells where M is non-zero only (none: +inf / -inf).  nprob > 1: over nprob such matrices,
// `bstride` elements apart (no selector); rag (a ragged batch's table): matrix b's first rag[b].rows rows only, or with
// rag_cols its first rag[b].rows columns (a ragged NMFD batch: the real positions of every line of the sliding axis).
int matrix_minmax(const void* V, int vdtype, int64_t rows, int64_t cols, int64_t ld, float* scratch2048, float* mm,
                  cudaStream_t st, CellSel M = CellSel{}, int64_t nprob = 1, int64_t bstride = 0,
                  const RaggedProblem* rag = nullptr, bool rag_cols = false);
// *out = sum of n doubles in fixed order (single block).  nprob > 1: out[b] = the sum of p[b n, (b + 1) n), one block per
// problem, in the same order; a problem whose `active` flag is 0 keeps its out[b].  rag (a ragged batch's table): problem
// b's run is its own rag[b].loss_n loss partials at rag[b].loss_part (n is not read).
int sum_partials(const double* p, int n, double* out, cudaStream_t st, int64_t nprob = 1, const uint8_t* active = nullptr,
                 const RaggedProblem* rag = nullptr);

// ard.cu -----------------------------------------------------------------------------------
// The relevance update of an l1-ARD fit (Tan and Fevotte 2013): with sW[k] and sH[k] the sums of component k of W (rows_w
// x R x inner_w) and H (rows_h x R x inner_h), each by factor_colsum in its fixed order (through `scratch`),
//   lambda[k] = (sW[k] + sH[k] + b) / c  (in double, stored as fp32),  pen[k] = phi / lambda[k]  (double, stored as fp32),
// and, unless `first`, *change = max_k |lambda[k] - old lambda[k]| / old lambda[k] (0 when `first`).  state: the ARD
// buffer, ard_state_floats(R) floats laid out [sW R | sH R | lambda R | pen R | change 1].  No float atomics: deterministic.
int64_t ard_state_floats(int R);
int ard_update(const float* W, int64_t rows_w, int64_t inner_w, const float* H, int64_t rows_h, int64_t inner_h, int R,
               double b, double c, double phi, bool first, float* scratch, int64_t scratch_floats, float* state,
               cudaStream_t st);

// project.cu -------------------------------------------------------------------------------
// Hoyer's projection (nmf.py:21-49) of every slice x[:, j, :] of x viewed as (outer, D, inner) onto {v >= 0, |v|_1 = k1[j],
// |v|_2^2 = k2[j]}, in place; zeroed_ws: D * outer * inner bytes of scratch.
int hoyer_project(float* x, int64_t outer, int D, int64_t inner, const float* k1, const float* k2,
                  unsigned char* zeroed_ws, cudaStream_t st);

// sparse_nmf.cu ----------------------------------------------------------------------------
// Sparse-target NMF (nmf.py:603-638): update terms at the non-zeros of V only, one warp per compressed segment.  The numerator
// of any beta > 0; the denominators of beta 1 (factor_colsum) and 2 (Gram) are below, of other beta simt_nmf_contract_den.
int sparse_numerator(const int64_t* ptr, const int64_t* idx, const float* val, const float* Fself, const float* Fother,
                     int R, int64_t nseg, double beta, float* out, cudaStream_t st);
int sparse_rows_times_gram(const float* F, const float* G, int64_t rows, int R, float* out, cudaStream_t st);
int sparse_loss(const int64_t* crow, const int64_t* col, const float* val, const float* H, const float* W, int R, int64_t N,
                double beta, const float* pos_a, const float* pos_b, double v_norm, double* loss_part, double* loss_dev,
                cudaStream_t st);
// beta != 1, 2 (the numerator: sparse_numerator): loss_dev = V_norm - neg from the gather over the CSR form + (sum of the npos
// V-free pos_part from simt_nmf_pow_sum) / beta
int sparse_beta_loss(const int64_t* crow, const int64_t* col, const float* val, const float* H, const float* W, int R,
                     int64_t N, double beta, const double* pos_part, int npos, double* loss_part, double* loss_dev,
                     cudaStream_t st);
// Observed cells of a masked fit (the stored entries, zeros included), every beta: both raw terms of one factor's update in one
// gather per segment (num, den: nseg x R), and loss_dev = beta_div(WH[obs], V[obs]) over the CSR form (loss_part: one double
// per gather block over the N rows).  wt (optional): one weight per stored entry, in the order of val -- each entry's
// terms and loss term are multiplied by it.
int observed_terms(const int64_t* ptr, const int64_t* idx, const float* val, const float* Fself, const float* Fother, int R,
                   int64_t nseg, double beta, float* num, float* den, cudaStream_t st, const float* wt = nullptr);
int observed_loss(const int64_t* crow, const int64_t* col, const float* val, const float* H, const float* W, int R, int64_t N,
                  double beta, double* loss_part, double* loss_dev, cudaStream_t st, const float* wt = nullptr);
// launch plans (host only): rank floats per lane; blocks over nseg segments / rows (the loss: N, its partials); Gram rows per
// block and blocks over `rows` rows; Gram passes of 4096 pairs
int sparse_rpl(int R);
int64_t sparse_gather_blocks(int64_t nseg);
void sparse_gram_plan(int64_t rows, int64_t* rpb, int* nb);
int sparse_gram_passes(int R);

// sparse_plca.cu ---------------------------------------------------------------------------
// Sparse-target PLCA (nmfb200_plca_sparse_*): V (N x C) in both compressed forms, borrowed -- CSR (crow, col, val: the
// normalised values) and CSC (ccol, row) with perm[e] the CSR position of the e-th CSC entry.
struct SparsePlcaTarget {
  const int64_t *crow = nullptr, *col = nullptr, *ccol = nullptr, *row = nullptr, *perm = nullptr;
  const float* val = nullptr;
  int64_t N = 0, C = 0;
  int R = 0;
};
// workspace: P (nnz floats), loss_part (sparse_plca_loss_parts doubles), cs_part (the two column sums' partials,
// sparse_plca_colsum_parts(C, R) + sparse_plca_colsum_parts(N, R) doubles)
struct SparsePlcaWork {
  float* P = nullptr;
  double* loss_part = nullptr;
  double* cs_part = nullptr;
};
void sparse_plca_colsum_plan(int64_t rows, int64_t* rpb, int* nb);
int64_t sparse_plca_loss_parts(int64_t N);
int64_t sparse_plca_colsum_parts(int64_t rows, int R);
// dW (C x R) and dHz (N x R) of one EM step at (W, Hz), each skipped when null; loss_dev (optional) the KL loss of norm q
int sparse_plca_terms(const SparsePlcaTarget& t, const SparsePlcaWork& ws, const float* W, const float* Hz, float* dW,
                      float* dHz, float norm, double* loss_dev, cudaStream_t st);

// plca_em.cu -------------------------------------------------------------------------------
// The EM step of nprob PLCA problems (nmfb200_plca_iterate), one block per problem: W (wrows, R, winner) and H, Hz (hrows, R,
// hinner) per problem back to back, Z (R) per problem; dW / dHz the raw numerators in the factors' shapes; aW / aH / aZ the
// alphas in the factors' shapes (null: 1); `flags` NMFB200_PLCA_TRAIN_*; buf: nprob x plca_em_buf_floats of scratch.
// rag (a ragged PLCA batch's table, hinner 1): problem p's H side -- H, Hz, dHz and aH -- is its first rag[p].rows of the
// hrows rows, each step summed as a batch of that many rows sums it; the rows past them are neither read nor written.
int plca_em(int64_t nprob, int64_t wrows, int64_t winner, int64_t hrows, int64_t hinner, int R, float* W, float* H, float* Z,
            float* Hz, const float* dW, const float* dHz, const float* aW, const float* aH, const float* aZ, int flags,
            float* buf, const uint8_t* active, const RaggedProblem* rag, cudaStream_t st);
int64_t plca_em_buf_floats(int R, int64_t w_inner, int64_t h_inner);

// nmfd.cu ----------------------------------------------------------------------------------
// L, T, Lin are the sizes along the LAST (contiguous) axis; NMF2D / NMF3D (nmf.py:782-942) add up to two outer axes of the
// target (X1, X2), of the kernel (T1, T2) and of H (X - T + 1).  The outer axes are loops around the same sliding GEMMs.
struct NmfdShape {
  int B, C, L, R, T, Lin;
  int X1 = 1, X2 = 1, T1 = 1, T2 = 1;
  __host__ __device__ int J1() const { return X1 - T1 + 1; }
  __host__ __device__ int J2() const { return X2 - T2 + 1; }
  __host__ __device__ int64_t v_inner() const { return (int64_t)X1 * X2 * L; }        // target elements per (b, c)
  __host__ __device__ int64_t w_inner() const { return (int64_t)T1 * T2 * T; }        // kernel elements per (c, r)
  __host__ __device__ int64_t h_inner() const { return (int64_t)J1() * J2() * Lin; }  // activation elements per (b, r)
  __host__ __device__ bool one_d() const { return X1 == 1 && X2 == 1 && T1 == 1 && T2 == 1; }
};
// WH = conv(H, W); writes Pn (and Pp when beta != 1) (B,C,L) or, when loss_blocks != nullptr,
// reduces beta_div(WH, V) instead.  M (optional selector in V's layout): Pn = Pp = 0 at the missing cells and V is not read
// there, Pp is written at every beta (beta 1: Pp = M as 0 / 1), and the loss skips them; a weight selector also multiplies
// Pn, Pp and the loss term by the cell's weight (beta 1: Pp = the weight).
// bt (no selector; nmfb200_nmfnd_batched_create): bt.n problems of shape s in the same launches, problem b with its target
// at V + b bt.v (0: one shared target) and its W, H, Pn, Pp in the b-th block of (bt.n, ...) storages; loss_dev[b] from its
// own run of partials summed in the single problem's order.  Problems whose bt.active flag is 0 are skipped: their factors'
// terms and loss_dev slots are left as they are.  The kernels derive bt.f / bt.g / bt.p from s; the caller's are not read.
// bt.rag (a ragged batch, s its padded shape): problem b runs the plan of its own length rag[b].rows along the sliding
// axis, reads V and H in their padded layouts up to that length and writes its tiles and loss partials at its own offsets
// (RaggedProblem); so do nmfd_wgrad and nmfd_dgrad, nsplit then the largest problem's.
int nmfd_recon_phi(const NmfdShape& s, const void* V, int vdtype, const float* W, const float* H, double beta,
                   float* Pn, float* Pp, double* loss_blocks, int max_blocks, double* loss_dev,
                   cudaStream_t st, CellSel M = CellSel{}, const Batch& bt = Batch{});
// The kPlcaFill mode of nmfd_recon_phi (one problem, fp32 V, uint8 mask M in V's layout, rank <= 256): Pn = M V / (WH + eps)
// and Pp = (1 - M) WH / (WH + eps) in V's layout, and *qobs_dev = the sum of WH over the observed cells, from one double
// partial per block of all its launches (nmfd_max_blocks, at most max_blocks) summed in a fixed order.
int nmfd_plca_fill(const NmfdShape& s, const float* V, const float* W, const float* H, float* Pn, float* Pp,
                   const uint8_t* M, double* part, int max_blocks, double* qobs_dev, cudaStream_t st);
// batch elements per launch of the kernels that put the batch on grid.z (fp32 recon / dgrad, tensor-core recon / dgrad)
static inline int64_t nmfd_batch_slice(int64_t B) { return B < kMaxGridYZ ? B : kMaxGridYZ; }
// loss partials of nmfd_recon_phi: one per block of all its launches
int64_t nmfd_max_blocks(const NmfdShape& s);
// out[c,r,t] = sum_{b,x} G[b,c,x] H[b,r,x-t]   (x, t multi-indices over up to three axes)
// bt (as nmfd_recon_phi's): out[split][problem][C,R,T], each problem's lines in the single problem's splits
int nmfd_wgrad(const NmfdShape& s, const float* G, const float* H, float* out, int nsplit, cudaStream_t st,
               const Batch& bt = Batch{});   // out[split][C,R,T]
int nmfd_wgrad_nsplit(const NmfdShape& s);
// out[split][b,r,j] = sum_{c in split, t} W[c,r,t] G[b,c,j+t]   (j, t multi-indices)
// bt (as nmfd_recon_phi's): out[split][problem][B,R,J]
int nmfd_dgrad(const NmfdShape& s, const float* G, const float* W, float* out, int nsplit, cudaStream_t st,
               const Batch& bt = Batch{});
int nmfd_dgrad_nsplit(const NmfdShape& s);
// wgrad's block plan (nmfd.cu): row tile MT of channels, TP = roundup(min(T, 64), 4) offsets of NR components for NO outer
// kernel offsets per block; NTT x NRG x NOG column blocks
struct WgradPlan { int mt, tp, nr, no, ntt, nrg, nog; };
// what nmfd_recon_phi / nmfd_dgrad / nmfd_wgrad launch for this shape, with the splits the library uses
// (recon and dgrad grids are per launch: batches beyond grid.z take ceil(B / z) launches)
struct NmfdPlan {
  int recon_mt; Grid3 recon_grid; int dgrad_mt, dgrad_nsplit; Grid3 dgrad_grid; WgradPlan wgrad; int wgrad_nsplit;
  Grid3 wgrad_grid;
};
Grid3 wgrad_grid(const NmfdShape& s, const WgradPlan& p, int nsplit);
void nmfd_plan(const NmfdShape& s, NmfdPlan* p);

}  // namespace nmfb200
