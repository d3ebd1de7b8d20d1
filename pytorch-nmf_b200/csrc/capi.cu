// C ABI of libnmf_b200 (see include/nmf_b200.h): context management and the per-update call graphs.
#include "../../include/nmf_b200.h"

#include <algorithm>
#include <cmath>
#include <atomic>
#include <functional>
#include <new>
#include <vector>

#include "common.cuh"
#include "tc_nmf.cuh"
#include "tc_nmfd.cuh"

namespace nmfb200 {
static thread_local std::string g_err;
static std::atomic<int64_t> g_launches{0};
void set_error(const std::string& msg) { g_err = msg; }
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
}  // namespace nmfb200

using namespace nmfb200;

// NmfBatch / NmfdBatch: a batch of NMF / of NMFD, NMF2D, NMF3D problems; PlcaSparse: served by its own calls only
enum class CtxKind { Nmf, Nmfd, NmfBatch, NmfdBatch, PlcaSparse };

// What the last successful set_target* registered.  Observed: the compressed forms hold the observed cells of a masked fit,
// and every beta fits beta_div(WH[obs], V[obs]) on the observed-cell gathers.
enum class TargetForm { None, Dense, Sparse, SparseAnyBeta, Observed };

// A sparse target, borrowed: CSR (rows of V) and CSC (= CSR of V^T) forms; an observed target's entry weights in CSR / CSC
// order (none: unweighted); V_norm of nmf.py:161-170 (beta 1 / 2); sparse PLCA's CSR position of each CSC entry; the
// stored entries' count (set by set_sparse_target)
struct SparseTarget {            // members in the order of the set_target_sparse* arguments
  const int64_t* crow = nullptr; const int64_t* col = nullptr; const float* val = nullptr;
  const int64_t* ccol = nullptr; const int64_t* row = nullptr; const float* val_t = nullptr;
  const float *wt = nullptr, *wt_t = nullptr;
  double vnorm_kl = 0.0, vnorm_eu = 0.0;
  const int64_t* perm = nullptr;
  int64_t nnz = 0;
};

// A device buffer a context owns: `n` elements of T, freed with the context (an empty one makes no CUDA call)
template <class T>
struct DevBuf {
  T* p = nullptr;
  int64_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  operator T*() const { return p; }
  // at least `count` elements: allocated on first need, or grown (dropping the contents)
  cudaError_t ensure(int64_t count) {
    if (p && n >= count) return cudaSuccess;
    if (p) { cudaFree(p); p = nullptr; n = 0; }
    const cudaError_t e = cudaMalloc(&p, (size_t)count * sizeof(T));
    if (e == cudaSuccess) n = count;
    return e;
  }
};

struct nmfb200_ctx {
  CtxKind kind = CtxKind::Nmf;
  int device = 0;
  int precision = NMFB200_PREC_F32;
  bool auto_mode = false;   // precision AUTO: the tensor-core path is used only where it is known to hold the parity bar
  bool tc_off = false;      // AUTO found the target outside the fp16 operand range: fp32 CUDA-core kernels instead
  int64_t N = 0, C = 0, R = 0;
  // a batch: nprob problems of the shape (N, C, R) or d, their targets bstride elements apart (0: one shared
  // target), factors and partial slabs back to back; `active` (borrowed, nprob device bytes, null: all) flags the problems
  // that run
  int64_t nprob = 1, bstride = 0;
  const uint8_t* active = nullptr;
  // a ragged batch of NMF problems (nmfb200_nmf_batched_create_ragged): each problem's plan (device, nprob of them)
  // and the grid x of each RaggedLaunch, the sum of the problems' blocks
  DevBuf<RaggedProblem> rag;
  int64_t rag_gx[4] = {0, 0, 0, 0};
  NmfdShape d{};
  const void* V = nullptr;        // the dense target, borrowed: vdtype (NMFB200_DTYPE_*) elements
  int vdtype = NMFB200_DTYPE_F32;
  int64_t ldv = 0;
  TargetForm form = TargetForm::None;
  SparseTarget sp;
  // nmfb200_set_mask / nmfb200_set_weight: the observed cells (uint8) or the cells' weights (fp32), V's shape, contiguous,
  // borrowed; cleared by every set_target*.  While set, every pass runs the selecting fp32 kernels and beta 1 takes its
  // denominators from the contraction, not the column sums.
  CellSel sel;
  // nmfb200_set_fixed_w: R bytes, non-zero for a component of W held at its value, borrowed; cleared by every set_target*.
  // While set, every call that writes W leaves those components unstored.
  const uint8_t* fixed_w = nullptr;
  // nmfb200_set_ard: automatic relevance determination is registered (`ard`), with its prior's b, c = n_W + n_H + a + 1 and
  // the dispersion phi; cleared by every set_target*.  ard_state (kept across registrations): ard_state_floats(R) floats,
  // [sW R | sH R | lambda R | pen R | change 1].  While set, every W and H update adds pen[k] to the denominators of
  // component k, and nmf_iterate runs the lambda update after each H update.
  bool ard = false;
  double ard_b = 0.0, ard_c = 0.0, ard_phi = 0.0;
  DevBuf<float> ard_state;
  // chunked partial numerators / denominators of the CUDA-core path; den (lazy) is sized like num
  DevBuf<float> num, den;
  int nslab[2] = {1, 1};          // partial slabs of the W / H terms: contraction chunks (NMF), wgrad / dgrad splits (NMFD)
  DevBuf<float> colsum;           // [2][R]: 0 = colsum(W), 1 = colsum(H)
  DevBuf<float> cs_scratch;
  DevBuf<double> loss_blocks;
  DevBuf<float> mm_scratch;       // kMmFloats: matrix_minmax's partials, then the target's min / max
  DevBuf<float> sp_den;           // max(N, C) x R: the reduced V-free denominator of an update at beta != 1, 2
  DevBuf<float> sp_gram;          // [2][R*R] (W^T W, H^T H) + per-block partials; also the Gram scratch of nmfb200_nmf_cd_*
  DevBuf<float> obs_r;            // nmfb200_nmf_observed_cd_*: one residual per observed entry (R > 32 only)
  DevBuf<double> sp_loss_part;
  // NMFD: the ratio tiles, Pp (lazy) sized like Pn (a batch: every problem's, back to back)
  DevBuf<float> Pn, Pp;
  // nmfb200_plca_masked_terms on NMF: one q_O partial per block of the fp32 contraction (grown on demand)
  DevBuf<double> qobs_part;
  // tensor-core path state (tc_nmf.cu / tc_nmfd.cu)
  TcState* tc = nullptr;
  TcNmfdState* tcd = nullptr;
  // sparse-target PLCA: the workspace of SparsePlcaWork and its nnz
  DevBuf<float> spl_P;
  DevBuf<double> spl_loss_part, spl_cs_part;
  int64_t spl_nnz = 0;
};

namespace {

int fail(int code, const std::string& msg) { set_error(msg); return code; }

// Every entry point runs on the context's device and leaves the calling thread's current device as it found it
// (a fit() on a module living on cuda:1 must not redirect the caller's later "cuda" allocations).
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess) { ok = false; return; }
    if (cur != dev) {
      if (cudaSetDevice(dev) != cudaSuccess) { ok = false; return; }
      prev = cur;
    }
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// A set of context kinds, one bit per kind: what an entry point serves
template <class... K>
constexpr unsigned kinds(K... k) { return ((1u << static_cast<int>(k)) | ...); }
constexpr unsigned kDenseModels = kinds(CtxKind::Nmf, CtxKind::Nmfd, CtxKind::NmfBatch, CtxKind::NmfdBatch);
constexpr unsigned kDenseNmf = kinds(CtxKind::Nmf, CtxKind::NmfBatch);
inline bool is_nmfd(const nmfb200_ctx* c) { return c->kind == CtxKind::Nmfd || c->kind == CtxKind::NmfdBatch; }
inline bool is_batch(const nmfb200_ctx* c) { return c->kind == CtxKind::NmfBatch || c->kind == CtxKind::NmfdBatch; }
inline bool has_target(const nmfb200_ctx* c) { return c->form != TargetForm::None; }
// a compressed target (c->sp): the dense kernels are out of play
inline bool is_sparse(const nmfb200_ctx* c) { return has_target(c) && c->form != TargetForm::Dense; }
#define CTX_GUARD(ctx, kind_set)                                                    \
  if (!(ctx)) return fail(NMFB200_ERR_INVALID, "null context");                     \
  if (!((kind_set) & kinds((ctx)->kind)))                                           \
    return fail(NMFB200_ERR_INVALID, "wrong context kind");                         \
  DeviceGuard _dev_guard((ctx)->device);                                            \
  if (!_dev_guard.ok) return fail(NMFB200_ERR_CUDA, "cannot select the context's device");
#define TARGET_GUARD(ctx) \
  if (!has_target(ctx)) return fail(NMFB200_ERR_STATE, "set_target has not been called");

// mm_scratch: kMmPartials per-block partials of matrix_minmax, then the target's min / max
constexpr int kMmPartials = 2048;
constexpr int kMmFloats = kMmPartials + 2;

// Chunks of the contracted dimension of the fp32 contraction.  Above rank 256 the grid already holds one CTA per rank block
// (simt_rank_blocks) for every row block and chunk: counting them keeps the nch x rows x R partial slabs from growing with
// the blocks.
// rank blocks of 256 components ride on grid z of the contraction and grid y of the column sum
constexpr int64_t kMaxRank = kMaxGridYZ * 256;
constexpr const char* kMaxRankMsg = "rank must be at most 65535 x 256 = 16776960";

int chunks_for(int64_t rows, int64_t cols, int64_t R) {
  int64_t rb = ceil_div(rows, 64) * simt_rank_blocks((int)R), tiles = ceil_div(cols, 64);
  int64_t want = ceil_div(132 * 4, rb);      // a few waves over the 132 SMs of an H100
  if (want > tiles) want = tiles;
  if (want > 32) want = 32;
  if (want < 1) want = 1;
  return (int)want;
}

// sp_gram's floats: the two R x R Gram matrices and sparse_gram's block partials (R <= 256).  A batch of P problems:
// [2][P][R^2], then each problem's partials on its own Gram plan, P x max(nb(N), nb(C)) R^2 (sparse_gram_plan), not P x the
// fixed 128 R^2.
int64_t gram_floats(const nmfb200_ctx* c) {
  const int64_t R = c->R;
  if (!is_batch(c)) return 2 * R * R + sparse_gram_part_floats((int)R);
  int64_t rpb;
  int nb_n, nb_c;
  sparse_gram_plan(c->N, &rpb, &nb_n);
  sparse_gram_plan(c->C, &rpb, &nb_c);
  return c->nprob * (2 + (int64_t)(nb_n > nb_c ? nb_n : nb_c)) * R * R;
}

void free_ctx(nmfb200_ctx* c) {
  if (!c) return;
  DeviceGuard guard(c->device);
  if (c->tc) tc_destroy(c->tc);
  if (c->tcd) tc_nmfd_destroy(c->tcd);
  delete c;
}

// A context's shape and what it allocates at create: the partial slabs (num), the column-sum scratch, the loss partials and
// NMFD's ratio tile Pn (0: none); a ragged batch's per-problem plans and the grid x of each RaggedLaunch.  nslab: the partial
// slabs of the W / H terms (contraction chunks of NMF, wgrad / dgrad splits of NMFD).
struct CtxPlan {
  int64_t N = 0, C = 0, R = 0, nprob = 1;
  NmfdShape d{};
  int nslab[2] = {1, 1};
  int64_t part_floats = 0, cs_scratch_floats = 0, loss_blocks = 0, pn_floats = 0;
  std::vector<RaggedProblem> rag;
  int64_t rag_gx[4] = {0, 0, 0, 0};
};

// P NMF problems of one shape: each problem's plan is the single problem's (P = 1), its workspace after the previous ones'
CtxPlan plan_nmf(int64_t N, int64_t C, int64_t R, int64_t P) {
  CtxPlan p{N, C, R, P};
  p.nslab[0] = chunks_for(C, N, R);
  p.nslab[1] = chunks_for(N, C, R);
  p.part_floats = std::max((int64_t)p.nslab[0] * C * R, (int64_t)p.nslab[1] * N * R) * P;
  p.cs_scratch_floats = colsum_scratch_floats(std::max(N, C), (int)R, 1) * P;
  p.loss_blocks = simt_nmf_max_blocks(N, C) * P;
  return p;
}

// A ragged batch of B NMF problems: each problem's single-problem plan along its own length, its blocks after the previous
// problems' on grid x and its workspace after theirs
int plan_nmf_ragged(int64_t B, int64_t N, int64_t C, int64_t R, const int64_t* lengths, CtxPlan* out) {
  CtxPlan plan{N, C, R, B};
  plan.rag.resize(B);
  int64_t* gx = plan.rag_gx;
  int64_t cs = 0;
  const int64_t w_blocks = ceil_div(C, 64);
  for (int64_t b = 0; b < B; ++b) {
    const int64_t L = lengths[b];
    if (L < 1 || L > N)
      return fail(NMFB200_ERR_INVALID, "lengths[" + std::to_string(b) + "] = " + std::to_string(L) + " is outside [1, N]");
    RaggedProblem& p = plan.rag[b];
    p.rows = L;
    p.nch[0] = chunks_for(C, L, R);
    p.nch[1] = chunks_for(L, C, R);
    SimtNmfPlan sp;
    simt_nmf_plan(L, C, (int)R, p.nch[1], &sp);
    p.loss_chunks = sp.loss_chunks;
    p.cs_blocks = (int)colsum_scratch_floats(L, 1, 1);
    const int64_t blocks[4] = {w_blocks * p.nch[0], ceil_div(L, 64) * p.nch[1], ceil_div(L, 64) * p.loss_chunks, p.cs_blocks};
    for (int k = 0; k < 4; ++k) { p.x0[k] = gx[k]; gx[k] += blocks[k]; }
    p.part = plan.part_floats; p.loss_part = plan.loss_blocks; p.cs_part = cs; p.loss_n = blocks[2];
    plan.part_floats += std::max((int64_t)p.nch[0] * C * R, (int64_t)p.nch[1] * L * R);
    plan.loss_blocks += blocks[2];
    cs += p.cs_blocks * R;
    // checked after every problem, so no sum can overflow int64 first
    if (gx[0] > kMaxGridX || gx[1] > kMaxGridX || gx[2] > kMaxGridX || gx[3] > kMaxGridX)
      return fail(NMFB200_ERR_INVALID, "ragged batch: the problems' blocks of one launch pass grid x (2^31 - 1)");
    if (plan.loss_blocks > INT32_MAX) return fail(NMFB200_ERR_INVALID, "ragged batch: loss partials must be below 2^31");
  }
  // the launches every problem shares the shape of: the column sums of W, their final stage, the ratio stage
  if (colsum_scratch_floats(C, 1, 1) > kMaxGridX / B || ceil_div(R, 64) > kMaxGridX / B ||
      ceil_div(std::max(N, C) * R, 256) > kMaxGridX / B)
    return fail(NMFB200_ERR_INVALID, "batch too large for the launch grids");
  plan.nslab[0] = chunks_for(C, N, R);      // unused by the ragged launches: each problem's own counts are in its plan
  plan.nslab[1] = chunks_for(N, C, R);
  plan.cs_scratch_floats = std::max(cs, colsum_scratch_floats(C, (int)R, 1) * B);
  *out = std::move(plan);
  return 0;
}

// P NMFD / NMF2D / NMF3D problems of shape d: each problem's plan is the single problem's (P = 1), its workspace after the
// previous ones'
CtxPlan plan_nmfd(const NmfdShape& d, int64_t P) {
  const int64_t B = d.B, C = d.C, R = d.R;
  CtxPlan p{0, 0, R, P, d};
  p.nslab[0] = nmfd_wgrad_nsplit(d);
  p.nslab[1] = nmfd_dgrad_nsplit(d);
  p.part_floats = std::max((int64_t)p.nslab[0] * C * R * d.w_inner(), (int64_t)p.nslab[1] * B * R * d.h_inner()) * P;
  p.cs_scratch_floats =
      std::max(colsum_scratch_floats(C, (int)R, d.w_inner()), colsum_scratch_floats(B, (int)R, d.h_inner())) * P;
  p.loss_blocks = nmfd_max_blocks(d) * P;
  p.pn_floats = B * C * d.v_inner() * P;
  return p;
}

// A ragged batch of P NMFD / NMF2D / NMF3D problems of padded shape d: each problem's single-problem plan along its own
// length, its workspace after the previous problems'.  Every count is at most the padded shape's, which the batch's shape
// checks bound for P problems.
int plan_nmfd_ragged(const NmfdShape& d, int64_t P, const int64_t* lengths, CtxPlan* out) {
  const int64_t B = d.B, C = d.C, R = d.R;
  CtxPlan plan{0, 0, R, P, d};
  plan.rag.resize(P);
  plan.nslab[0] = nmfd_wgrad_nsplit(d);
  const int64_t wpart = (int64_t)plan.nslab[0] * C * R * d.w_inner();
  int64_t cs = 0;
  for (int64_t p = 0; p < P; ++p) {
    const int64_t L = lengths[p];
    if (L < d.T || L > d.L)
      return fail(NMFB200_ERR_INVALID, "lengths[" + std::to_string(p) + "] = " + std::to_string(L) + " is outside [" +
                                           std::to_string(d.T) + ", " + std::to_string(d.L) + "] (the last kernel and target sizes)");
    NmfdShape e = d;
    e.L = (int)L; e.Lin = (int)(L - d.T + 1);
    NmfdPlan np;
    nmfd_plan(e, &np);
    RaggedProblem& q = plan.rag[p];
    q.rows = L; q.lin = e.Lin;
    q.gx[0] = (int)np.recon_grid.x; q.gx[1] = (int)np.dgrad_grid.x;
    q.nch[0] = np.wgrad_nsplit; q.nch[1] = np.dgrad_nsplit;
    q.loss_n = nmfd_max_blocks(e);
    // the column sums of H at beta 1 as its single fit forms them: one partial per (clip, component) run, or the rows
    // blocking of a run of one element
    q.cs_blocks = (int)(e.h_inner() > 1 ? B : colsum_scratch_floats(B, 1, 1));
    q.pn = plan.pn_floats; q.part = plan.part_floats; q.loss_part = plan.loss_blocks; q.cs_part = cs;
    plan.nslab[1] = std::max(plan.nslab[1], np.dgrad_nsplit);    // the dgrad launch's grid y; each problem runs its own splits
    // every problem's tiles and slabs start 16-byte aligned: the ratio stage of W reads its slabs as float4 (update.cu:
    // apply_update_vec4_kernel) wherever the shape allows, and a dgrad slab may hold any number of floats
    plan.pn_floats += round_up(B * C * e.v_inner(), 4);
    plan.part_floats += round_up(std::max(wpart, (int64_t)np.dgrad_nsplit * B * R * e.h_inner()), 4);
    plan.loss_blocks += q.loss_n;
    cs += B * R;
  }
  plan.cs_scratch_floats = std::max(cs, colsum_scratch_floats(C, (int)R, d.w_inner()) * P);
  *out = std::move(plan);
  return 0;
}

// A refused create leaves *out null
int check_out(nmfb200_ctx** out) {
  if (!out) return fail(NMFB200_ERR_INVALID, "out is null");
  *out = nullptr;
  return 0;
}

// The one constructor of every context kind, once the create's own checks have passed: selects `device`, allocates a
// context of `kind` and plan's shape, lets `init` (if any) set or refuse the rest of it, allocates what the plan asks for and
// uploads a ragged batch's plans, then runs `finish` (if any: the kind's tensor-core state or workspace) under the same
// device guard.  On any failure it frees everything and leaves *out null.
using CtxStep = std::function<int(nmfb200_ctx*)>;
int create_ctx(nmfb200_ctx** out, int device, CtxKind kind, const CtxPlan& plan, const CtxStep& init = nullptr,
               const CtxStep& finish = nullptr) {
  DeviceGuard guard(device);
  if (!guard.ok) return fail(NMFB200_ERR_CUDA, "cannot select the requested device");
  nmfb200_ctx* c = new (std::nothrow) nmfb200_ctx();
  if (!c) return fail(NMFB200_ERR_INVALID, "out of host memory");
  c->kind = kind; c->device = device; c->N = plan.N; c->C = plan.C; c->R = plan.R; c->nprob = plan.nprob; c->d = plan.d;
  c->nslab[0] = plan.nslab[0]; c->nslab[1] = plan.nslab[1];
  for (int k = 0; k < 4; ++k) c->rag_gx[k] = plan.rag_gx[k];
  int rc = init ? init(c) : 0;
  if (rc == 0 && plan.part_floats) {                  // the dense models' workspace
    cudaError_t e = c->num.ensure(plan.part_floats);
    if (e == cudaSuccess) e = c->colsum.ensure(2 * c->R * c->nprob);
    if (e == cudaSuccess) e = c->cs_scratch.ensure(plan.cs_scratch_floats);
    if (e == cudaSuccess) e = c->loss_blocks.ensure(plan.loss_blocks);
    if (e == cudaSuccess) e = c->mm_scratch.ensure(kMmFloats);
    if (e == cudaSuccess && plan.pn_floats) e = c->Pn.ensure(plan.pn_floats);
    if (e != cudaSuccess) rc = fail(NMFB200_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
  }
  if (rc == 0 && !plan.rag.empty()) {
    cudaError_t e = c->rag.ensure((int64_t)plan.rag.size());
    if (e == cudaSuccess)
      e = cudaMemcpy(c->rag, plan.rag.data(), plan.rag.size() * sizeof(RaggedProblem), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) rc = fail(NMFB200_ERR_CUDA, std::string("ragged batch plans: ") + cudaGetErrorString(e));
  }
  if (rc == 0 && finish) rc = finish(c);
  if (rc) { free_ctx(c); return rc; }
  *out = c;
  return 0;
}

// beta 1 without a mask: the denominator is the column sum of the other factor (nmf.py:122-131).  A masked or weighted fit
// takes it from the second backward pass, M G, like every other beta.
bool kl_colsum(const nmfb200_ctx* c, double beta) { return beta == 1.0 && !c->sel && c->form != TargetForm::Observed; }

// Whether the context's own tensor-core kernels (c->tc: NMF, c->tcd: NMFD / NMF2D / NMF3D) serve this beta.
bool use_tc(const nmfb200_ctx* c, double beta) {
  if (c->tc_off || c->sel) return false;
  if (c->tc) return tc_supports_beta(c->tc, beta);
  return c->tcd != nullptr && tc_nmfd_supported(c->d, beta);
}

// A pass outside the tensor-core state changed W (w) and / or H (h), or read them: NMF rebuilds the operand copies of the
// changed factors on their next use, NMFD everything it derived from either.
void mark_stale(nmfb200_ctx* c, bool w, bool h) {
  if (c->tc) tc_mark_dirty(c->tc, w, h);
  if (c->tcd) tc_nmfd_mark_dirty(c->tcd);
}

// One factor (which = 0: W, 1: H) and the other one: `rows` rows of R components x `inner` elements.  NMF: W is C x R and
// H is N x R; NMFD / NMF2D / NMF3D: W is C x R x w_inner and H is B x R x h_inner.
struct FactorDims { int64_t rows, inner, other_rows, other_inner; };
FactorDims factor_dims(const nmfb200_ctx* c, int which) {
  const NmfdShape& d = c->d;
  const FactorDims w = !is_nmfd(c) ? FactorDims{c->C, 1, c->N, 1} : FactorDims{d.C, d.w_inner(), d.B, d.h_inner()};
  return which == 0 ? w : FactorDims{w.other_rows, w.other_inner, w.rows, w.inner};
}

// The ratio stage's view of one factor's terms: its rows x R x inner elements, summed over `nchunks` slabs of that layout.
// A batch: the problems' factors back to back, each slab holding every problem's partials in that order.
ApplyArgs factor_view(const nmfb200_ctx* c, int which, int nchunks) {
  const FactorDims f = factor_dims(c, which);
  ApplyArgs a{};
  a.R = (int)c->R; a.inner = f.inner; a.rowlen = c->R * f.inner; a.ldp = a.rowlen;
  a.numel = f.rows * a.rowlen * c->nprob; a.chunk_stride = a.numel; a.nchunks = nchunks;
  if (is_batch(c)) { a.prob_numel = f.rows * a.rowlen; a.active = c->active; }
  if (c->rag) { a.rag = c->rag; a.rag_launch = which == 0 ? kRagW : kRagH; }
  if (c->rag && is_nmfd(c) && which == 1) a.line = c->d.Lin;      // a ragged NMFD batch's H: padding inside every line
  return a;
}

// The problems of one launch (kRagW / kRagH: the contraction of W / H, kRagLoss: the loss): the NMFD kernels take their
// strides from the shape; an NMF batch's F / G factors and partial slabs of problem b (slab layout [chunk][problem][rows][R],
// the loss: F = H, no slabs), and a ragged batch's launch and grid x.  One NMF problem: Batch{}, the single-problem kernels.
Batch launch_batch(const nmfb200_ctx* c, RaggedLaunch launch) {
  Batch bt;
  if (is_nmfd(c)) {
    bt = Batch{c->nprob, c->bstride, 0, 0, 0, c->active};
    bt.rag = c->rag;
    return bt;
  }
  if (!is_batch(c)) return bt;
  const FactorDims f = factor_dims(c, launch == kRagW ? 0 : 1);
  bt = Batch{c->nprob, c->bstride, f.rows * c->R, f.other_rows * c->R, launch == kRagLoss ? 0 : f.rows * c->R, c->active};
  if (c->rag) { bt.rag = c->rag; bt.rag_launch = launch; bt.rag_gx = c->rag_gx[launch]; }
  return bt;
}

// What every dense set_target checks of the target's element type and pointer (the kernels load single elements: element
// alignment is all they need).
int check_target(const void* V, int dtype) {
  if (!V) return fail(NMFB200_ERR_INVALID, "null target");
  if (dtype != NMFB200_DTYPE_F32 && dtype != NMFB200_DTYPE_F16 && dtype != NMFB200_DTYPE_BF16)
    return fail(NMFB200_ERR_INVALID, "unknown target dtype " + std::to_string(dtype) +
                                         " (NMFB200_DTYPE_F32 = 0, NMFB200_DTYPE_F16 = 1, NMFB200_DTYPE_BF16 = 2)");
  const int size = vdtype_size(dtype);
  if (reinterpret_cast<uintptr_t>(V) % size)
    return fail(NMFB200_ERR_INVALID, "target pointer is not aligned to its element size (" + std::to_string(size) + " bytes)");
  return 0;
}

// The one place a set_target* changes the target, once its checks and allocations have passed: a call refused before it
// leaves the context as it was.  A new target drops the mask or weight, the fixed components of W and the ARD registration;
// a sparse one takes the tensor cores out of play.
void commit_target(nmfb200_ctx* c, TargetForm form, const void* V, int vdtype, int64_t ldv, int64_t bstride,
                   const SparseTarget& sp = SparseTarget{}) {
  c->form = form; c->V = V; c->vdtype = vdtype; c->ldv = ldv; c->bstride = bstride; c->sp = sp;
  c->sel = CellSel{};
  c->fixed_w = nullptr;
  c->ard = false;
  c->tc_off = form != TargetForm::Dense;
}

// AUTO keeps heavy-tailed targets (max / mean > 64: spectrogram-like, lognormal, ...) off the tensor cores.  Measured on the
// lognormal fixtures of tests/golden/reference_r2.npz (30 iterations, tolerance rtol 1e-3): f16 34x, f16_split 2x, f32 0.1x
// of the tolerance -- MU on such targets converges slowly and keeps the per-update operand rounding instead of averaging it
// out as it does on well-conditioned data (uniform-like targets: 0.17x after 200 iterations).  `vsum` is the sum of the
// target's `cells` elements; the max comes from set_target's matrix_minmax.  Synchronises.
int auto_off_if_heavy_tailed(nmfb200_ctx* ctx, double vsum, double cells, cudaStream_t st) {
  float mm[2] = {0.f, 0.f};
  NMF_CUDA_CHECK(cudaMemcpyAsync(mm, ctx->mm_scratch + kMmPartials, sizeof(mm), cudaMemcpyDeviceToHost, st));
  NMF_CUDA_CHECK(cudaStreamSynchronize(st));
  const double mean = vsum / cells;
  ctx->tc_off = !(mean > 0.0) || (double)mm[1] > 64.0 * mean;
  return 0;
}

// Synchronises `stream` and reports whether a kernel of this library aborted an internal wait (on the current device).
int check_health(void* stream) {
  int rc = tc_check_wait_abort((cudaStream_t)stream);
  if (rc == 0) rc = tc_nmfd_check_wait_abort();
  if (rc > 0) return fail(NMFB200_ERR_STATE, "a kernel aborted an internal barrier wait; results are invalid");
  if (rc < 0) return fail(NMFB200_ERR_CUDA, std::string("stream synchronize: ") + cudaGetErrorString(cudaGetLastError()));
  return 0;
}

// What the four sparse set_target calls of an NMF context share: the checks and the workspace of `form`, then the commit
int set_sparse_target(nmfb200_ctx* ctx, TargetForm form, int64_t nnz, const SparseTarget& sp, void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::Nmf));
  if (nnz < 0 || !sp.crow || !sp.ccol || (nnz > 0 && (!sp.col || !sp.val || !sp.row || !sp.val_t)))
    return fail(NMFB200_ERR_INVALID, "bad compressed sparse target");
  if (ctx->R > 256)
    return fail(NMFB200_ERR_INVALID, "rank > 256 is not supported by the sparse-target kernels (densify the target)");
  NMF_CUDA_CHECK(ctx->sp_gram.ensure(gram_floats(ctx)));
  NMF_CUDA_CHECK(ctx->sp_loss_part.ensure(sparse_gather_blocks(ctx->N)));
  if (form != TargetForm::Sparse)                          // the denominator of an update outside raw_terms
    NMF_CUDA_CHECK(ctx->den.ensure(ctx->num.n));
  if (form == TargetForm::SparseAnyBeta) NMF_CUDA_CHECK(ctx->sp_den.ensure(std::max(ctx->N, ctx->C) * ctx->R));
  SparseTarget t = sp;
  t.nnz = nnz;
  commit_target(ctx, form, nullptr, NMFB200_DTYPE_F32, 0, 0, t);
  if (form != TargetForm::Observed) return 0;
  // target_minmax: the observed values (none: +inf / -inf)
  return matrix_minmax(sp.val, NMFB200_DTYPE_F32, 1, nnz, nnz, ctx->mm_scratch, ctx->mm_scratch + kMmPartials,
                       (cudaStream_t)stream);
}
}  // namespace

extern "C" {

int nmfb200_abi_version(void) { return NMFB200_ABI_VERSION; }
#ifndef NMFB200_SRC_HASH
#define NMFB200_SRC_HASH "unstamped"
#endif
#define NMFB200_STR2(x) #x
#define NMFB200_STR(x) NMFB200_STR2(x)
const char* nmfb200_build_info(void) {
  return "src=" NMFB200_SRC_HASH " nvcc=" NMFB200_STR(__CUDACC_VER_MAJOR__) "." NMFB200_STR(__CUDACC_VER_MINOR__) "."
         NMFB200_STR(__CUDACC_VER_BUILD__) " arch=sm_90a built=" __DATE__ " " __TIME__;
}
const char* nmfb200_last_error(void) { return g_err.c_str(); }
int64_t nmfb200_launch_count(void) { return g_launches.load(); }

int nmfb200_ctx_check_health(nmfb200_ctx* ctx, void* stream) {
  if (!ctx) return fail(NMFB200_ERR_INVALID, "null context");
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return fail(NMFB200_ERR_CUDA, "cannot select the context's device");
  if (ctx->tc) {
    const int pr = tc_peer_check(ctx->tc, (cudaStream_t)stream);
    if (pr > 0) return fail(NMFB200_ERR_STATE, "a sharded W update gave up waiting for rank " + std::to_string(pr - 1) +
                                               "'s buffer; results are invalid");
    if (pr < 0) return fail(NMFB200_ERR_CUDA, "stream synchronize failed");
  }
  return check_health(stream);
}

int nmfb200_nmf_create(nmfb200_ctx** out, int device, int64_t N, int64_t C, int64_t R, int precision) {
  if (int rc = check_out(out)) return rc;
  if (N < 1 || C < 1 || R < 1) return fail(NMFB200_ERR_INVALID, "N, C, R must be positive");
  if (R > kMaxRank) return fail(NMFB200_ERR_INVALID, kMaxRankMsg);
  if (precision < NMFB200_PREC_AUTO || precision > NMFB200_PREC_F16_SPLIT)
    return fail(NMFB200_ERR_INVALID, "unknown precision mode");
  auto init = [&](nmfb200_ctx* c) {
    int resolved = precision;
    // AUTO: single-rounded fp16 operands hold the north-star parity (rtol 1e-3) once the ratio tile is kappa-centred;
    // the parity tests check it against the reference at the configuration shapes
    if (precision == NMFB200_PREC_AUTO) resolved = tc_shape_supported(N, C, R) ? NMFB200_PREC_F16 : NMFB200_PREC_F32;
    if (resolved != NMFB200_PREC_F32 && !tc_shape_supported(N, C, R))
      return fail(NMFB200_ERR_INVALID, "shape not supported by the tensor-core path (need R <= 128)");
    c->precision = resolved;
    c->auto_mode = precision == NMFB200_PREC_AUTO;
    return 0;
  };
  auto finish = [&](nmfb200_ctx* c) {
    if (c->precision == NMFB200_PREC_F32) return 0;
    return tc_create(&c->tc, device, N, C, R, c->precision == NMFB200_PREC_F16_SPLIT);
  };
  return create_ctx(out, device, CtxKind::Nmf, plan_nmf(N, C, R, 1), init, finish);
}

void nmfb200_destroy(nmfb200_ctx* ctx) { free_ctx(ctx); }

int nmfb200_precision(const nmfb200_ctx* ctx) {
  if (!ctx) return -100;
  return ctx->tc_off ? NMFB200_PREC_F32 : ctx->precision;
}

int nmfb200_precision_for_beta(const nmfb200_ctx* ctx, double beta) {
  if (!ctx) return -100;
  if (!use_tc(ctx, beta)) return NMFB200_PREC_F32;
  // NMF's beta != 1, 2 kernels read only the hi halves of the operand copies
  return (ctx->tc && (beta == 1.0 || beta == 2.0)) ? ctx->precision : NMFB200_PREC_F16;
}

int nmfb200_nmf_plan(int64_t N, int64_t C, int64_t R, int64_t* out, int n) {
  if (!out || n < NMFB200_NMF_PLAN_LEN) return fail(NMFB200_ERR_INVALID, "plan buffer too small");
  if (N < 1 || C < 1 || R < 1) return fail(NMFB200_ERR_INVALID, "N, C, R must be positive");
  if (R > kMaxRank) return fail(NMFB200_ERR_INVALID, kMaxRankMsg);
  const int nch_w = chunks_for(C, N, R), nch_h = chunks_for(N, C, R);
  SimtNmfPlan pw, ph;
  simt_nmf_plan(C, N, (int)R, nch_w, &pw);          // W update: F = W (C rows), contracted over the N rows of V
  simt_nmf_plan(N, C, (int)R, nch_h, &ph);          // H update, and the loss (F = H)
  const int64_t v[NMFB200_NMF_PLAN_LEN] = {nch_w, nch_h, pw.tiles_per_chunk, ph.tiles_per_chunk, ph.rb, ph.loss_chunks,
                                           ph.loss_tiles_per_chunk, colsum_scratch_floats(N, 1, 1),
                                           colsum_scratch_floats(C, 1, 1)};
  for (int i = 0; i < NMFB200_NMF_PLAN_LEN; ++i) out[i] = v[i];
  return 0;
}

int nmfb200_nmf_sparse_plan(int64_t N, int64_t C, int64_t R, int64_t* out, int n) {
  if (!out || n < NMFB200_SPARSE_PLAN_LEN) return fail(NMFB200_ERR_INVALID, "plan buffer too small");
  if (N < 1 || C < 1 || R < 1) return fail(NMFB200_ERR_INVALID, "N, C, R must be positive");
  if (R > 256) return fail(NMFB200_ERR_INVALID, "rank > 256 is not supported by the sparse-target kernels (densify the target)");
  int64_t rpb_n, rpb_c;
  int nb_n, nb_c;
  sparse_gram_plan(N, &rpb_n, &nb_n);               // H^T H: the W update's beta-2 denominator, the beta-2 loss
  sparse_gram_plan(C, &rpb_c, &nb_c);               // W^T W: the H update's, the loss
  const int64_t v[NMFB200_SPARSE_PLAN_LEN] = {sparse_rpl((int)R), sparse_gram_passes((int)R), rpb_n, nb_n, rpb_c, nb_c,
                                              sparse_gather_blocks(N), sparse_gather_blocks(C)};
  for (int i = 0; i < NMFB200_SPARSE_PLAN_LEN; ++i) out[i] = v[i];
  return 0;
}

int nmfb200_nmf_set_target(nmfb200_ctx* ctx, const void* V, int64_t ldv, int dtype, void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::Nmf));
  if (!V || ldv < ctx->C) return fail(NMFB200_ERR_INVALID, "bad target pointer / leading dimension");
  if (int rc = check_target(V, dtype)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  commit_target(ctx, TargetForm::Dense, V, dtype, ldv, 0);
  float* minmax = ctx->mm_scratch + kMmPartials;
  int rc = matrix_minmax(V, dtype, ctx->N, ctx->C, ldv, ctx->mm_scratch, minmax, st);
  if (rc) return rc;
  if (ctx->tc) {
    rc = tc_set_target(ctx->tc, V, dtype, ldv, minmax, st);
    if (rc) return rc;
    if (ctx->auto_mode) {
      // AUTO is conservative: the fp16 copy of V carries ONE power-of-two scale (max -> 2^14), so positive entries below
      // max * 2^-28 lose precision or vanish (power spectrograms span more than that).  Targets with more than a
      // negligible share of such entries run on the fp32 kernels; asking for "f16" / "f16_split" explicitly keeps the
      // tensor cores.
      unsigned long long lossy = 0;
      rc = tc_target_lossy(ctx->tc, &lossy, st);
      if (rc) return rc;
      // a handful of tiny entries in a 10^8-cell matrix carry no structure; a quiet row / band (>= 1e-6 of the cells) does
      ctx->tc_off = (double)lossy > 1e-6 * (double)ctx->N * (double)ctx->C;
      if (!ctx->tc_off) {       // ... and for heavy-tailed targets
        double vsum = 0.0;
        rc = tc_target_sum(ctx->tc, &vsum, st);
        if (rc) return rc;
        return auto_off_if_heavy_tailed(ctx, vsum, (double)ctx->N * (double)ctx->C, st);
      }
    }
  }
  return 0;
}

/* ---- batched NMF: B independent problems of one shape on the fp32 kernels ------------------------------------ */

int nmfb200_nmf_batched_create(nmfb200_ctx** out, int device, int64_t B, int64_t N, int64_t C, int64_t R) {
  if (int rc = check_out(out)) return rc;
  if (B < 1 || N < 1 || C < 1 || R < 1) return fail(NMFB200_ERR_INVALID, "B, N, C, R must be positive");
  if (R > 256) return fail(NMFB200_ERR_INVALID, "batched fits support rank <= 256");
  // the batch rides on grid x of every launch, the loss partials are counted in int
  if (ceil_div(std::max(N, C), 64) > kMaxGridX / B || (int64_t)simt_nmf_max_blocks(N, C) > INT32_MAX / B ||
      ceil_div(R, 64) > kMaxGridX / B)
    return fail(NMFB200_ERR_INVALID, "batch too large for the launch grids");
  return create_ctx(out, device, CtxKind::NmfBatch, plan_nmf(N, C, R, B));
}

int nmfb200_nmf_batched_create_ragged(nmfb200_ctx** out, int device, int64_t B, int64_t N, int64_t C, int64_t R,
                                      const int64_t* lengths) {
  if (int rc = check_out(out)) return rc;
  if (B < 1 || N < 1 || C < 1 || R < 1) return fail(NMFB200_ERR_INVALID, "B, N, C, R must be positive");
  if (R > 256) return fail(NMFB200_ERR_INVALID, "batched fits support rank <= 256");
  if (!lengths) return fail(NMFB200_ERR_INVALID, "lengths is null");
  if (B > kMaxGridX) return fail(NMFB200_ERR_INVALID, "ragged batch: B must be below 2^31 (one block per problem and launch)");
  CtxPlan plan;
  if (int rc = plan_nmf_ragged(B, N, C, R, lengths, &plan)) return rc;
  return create_ctx(out, device, CtxKind::NmfBatch, plan);
}

int nmfb200_nmf_batched_set_target(nmfb200_ctx* ctx, const void* V, int64_t ldv, int64_t batch_stride, int dtype,
                                   void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::NmfBatch));
  if (!V || ldv < ctx->C) return fail(NMFB200_ERR_INVALID, "bad target pointer / leading dimension");
  if (batch_stride != 0 && batch_stride < ctx->N * ldv)
    return fail(NMFB200_ERR_INVALID, "batch stride must be 0 (one shared target) or at least N x ldv");
  if (int rc = check_target(V, dtype)) return rc;
  commit_target(ctx, TargetForm::Dense, V, dtype, ldv, batch_stride);
  // a ragged batch: every problem's own rows, even of a shared target
  return matrix_minmax(V, dtype, ctx->N, ctx->C, ldv, ctx->mm_scratch, ctx->mm_scratch + kMmPartials, (cudaStream_t)stream,
                       CellSel{}, batch_stride || ctx->rag ? ctx->nprob : 1, batch_stride, ctx->rag);
}

namespace {
// nmfb200_nmf_batched_set_active / nmfb200_nmfd_batched_set_active on a batch of `kind`
int set_active(nmfb200_ctx* ctx, CtxKind kind, const uint8_t* active) {
  CTX_GUARD(ctx, kinds(kind));
  ctx->active = active;
  return 0;
}
}  // namespace

int nmfb200_nmf_batched_set_active(nmfb200_ctx* ctx, const uint8_t* active, void* stream) {
  (void)stream;
  return set_active(ctx, CtxKind::NmfBatch, active);
}

/* ---- sparse targets (beta 1 and 2): nmf.py:603-638 without the dense product ------------------------------ */

int nmfb200_nmf_set_target_sparse(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow, const int64_t* col, const float* val,
                                  const int64_t* ccol, const int64_t* row, const float* val_t, double v_norm_kl,
                                  double v_norm_eu, void* stream) {
  return set_sparse_target(ctx, TargetForm::Sparse, nnz,
                           SparseTarget{crow, col, val, ccol, row, val_t, nullptr, nullptr, v_norm_kl, v_norm_eu}, stream);
}

int nmfb200_nmf_set_target_sparse_any_beta(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow, const int64_t* col,
                                           const float* val, const int64_t* ccol, const int64_t* row, const float* val_t,
                                           double v_norm_kl, double v_norm_eu, void* stream) {
  return set_sparse_target(ctx, TargetForm::SparseAnyBeta, nnz,
                           SparseTarget{crow, col, val, ccol, row, val_t, nullptr, nullptr, v_norm_kl, v_norm_eu}, stream);
}

int nmfb200_nmf_set_target_observed(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow, const int64_t* col,
                                    const float* val, const int64_t* ccol, const int64_t* row, const float* val_t,
                                    void* stream) {
  return set_sparse_target(ctx, TargetForm::Observed, nnz, SparseTarget{crow, col, val, ccol, row, val_t}, stream);
}

int nmfb200_nmf_set_target_observed_weighted(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow, const int64_t* col,
                                             const float* val, const int64_t* ccol, const int64_t* row, const float* val_t,
                                             const float* wt, const float* wt_t, void* stream) {
  if (nnz > 0 && (!wt || !wt_t)) return fail(NMFB200_ERR_INVALID, "bad entry weights");
  return set_sparse_target(ctx, TargetForm::Observed, nnz, SparseTarget{crow, col, val, ccol, row, val_t, wt, wt_t}, stream);
}

/* ---- NMFD ------------------------------------------------------------------------------------ */

// One context type serves NMFD (one sliding axis) and NMF2D / NMF3D (the last axis slides, the outer ones are loops):
// vdims / kdims hold the target's and the kernel's sizes over the ndim convolved axes.
// The context's shape from the create arguments (validated): the outer axes right-aligned, X2 / T2 innermost of them.
static int nmfd_shape_of(int64_t B, int64_t C, int ndim, const int64_t* vdims, int64_t R, const int64_t* kdims, NmfdShape* d) {
  if (ndim < 1 || ndim > 3 || !vdims || !kdims) return fail(NMFB200_ERR_INVALID, "1 to 3 convolved axes are supported");
  int64_t X[3] = {1, 1, 1}, K[3] = {1, 1, 1};            // right-aligned: X[2] / K[2] is the last (sliding) axis
  for (int i = 0; i < ndim; ++i) { X[3 - ndim + i] = vdims[i]; K[3 - ndim + i] = kdims[i]; }
  const int64_t L = X[2], T = K[2];
  if (B < 1 || C < 1 || R < 1) return fail(NMFB200_ERR_INVALID, "bad NMFD sizes");
  for (int i = 0; i < 3; ++i)
    if (K[i] < 1 || X[i] < K[i]) return fail(NMFB200_ERR_INVALID, "bad NMFD sizes");
  if (R > 256) return fail(NMFB200_ERR_INVALID, "rank > 256 is not supported");
  if (B * C * X[0] * X[1] * L > (int64_t)1 << 40 || X[0] * X[1] * L > (int64_t)1 << 30 || K[0] * K[1] * T > (int64_t)1 << 24)
    return fail(NMFB200_ERR_INVALID, "NMFD target too large");
  // every size below is narrowed to int, and the kernels count in int: bound what they derive from it
  if (C > kMaxGridYZ * 64)
    return fail(NMFB200_ERR_INVALID, "NMFD supports at most 65535 x 64 = 4194240 channels (grid.y of the reconstruction)");
  if (B * (X[0] - K[0] + 1) * (X[1] - K[1] + 1) > INT32_MAX)
    return fail(NMFB200_ERR_INVALID, "NMFD batch x outer activation lines must be below 2^31 (the W gradient's line index)");
  if ((C > R ? C : R) * K[0] * K[1] > INT32_MAX)
    return fail(NMFB200_ERR_INVALID, "NMFD channels (or rank) x outer kernel offsets must be below 2^31 (the contraction index)");
  *d = NmfdShape{(int)B, (int)C, (int)L, (int)R, (int)T, (int)(L - T + 1)};
  d->X1 = (int)X[0]; d->X2 = (int)X[1]; d->T1 = (int)K[0]; d->T2 = (int)K[1];
  NmfdPlan p;
  nmfd_plan(*d, &p);
  if (!grid_fits(p.recon_grid) || !grid_fits(p.dgrad_grid) || !grid_fits(p.wgrad_grid))
    return fail(NMFB200_ERR_INVALID, "an NMFD grid of the fp32 kernels passes the CUDA grid limits");
  if (nmfd_max_blocks(*d) > INT32_MAX) return fail(NMFB200_ERR_INVALID, "NMFD loss partials must number below 2^31");
  return 0;
}

int nmfb200_nmfnd_create(nmfb200_ctx** out, int device, int64_t B, int64_t C, int ndim, const int64_t* vdims,
                         int64_t R, const int64_t* kdims, int precision) {
  if (int rc = check_out(out)) return rc;
  NmfdShape shape;
  if (int rc = nmfd_shape_of(B, C, ndim, vdims, R, kdims, &shape)) return rc;
  if (precision != NMFB200_PREC_AUTO && precision != NMFB200_PREC_F32 && precision != NMFB200_PREC_F16)
    return fail(NMFB200_ERR_INVALID, "NMFD precision must be auto, f32 or f16");
  // NMF2D / NMF3D take the tensor-core kernels only when asked for (f16); auto keeps them on the fp32 kernels
  const bool one_d = shape.one_d();
  TcNmfdPlan tc_plan;
  const char* tc_limit = (one_d || precision == NMFB200_PREC_F16) ? tc_nmfd_plan(shape, &tc_plan) : "";
  if (precision == NMFB200_PREC_F16 && tc_limit) return fail(NMFB200_ERR_INVALID, tc_limit);
  auto finish = [&](nmfb200_ctx* c) {
    c->precision = precision == NMFB200_PREC_F32 ? NMFB200_PREC_F32 : NMFB200_PREC_F16;
    c->auto_mode = precision == NMFB200_PREC_AUTO;
    if (c->precision == NMFB200_PREC_F32 || tc_limit) return 0;    // NMFD at auto / f16, NMF2D / NMF3D at f16
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess && prop.major == 9)
      return tc_nmfd_create(&c->tcd, c->d);            // beta = 1 runs as wgmma sliding GEMMs (tc_nmfd.cu)
    if (precision == NMFB200_PREC_F16) return fail(NMFB200_ERR_INVALID, "the tensor-core NMFD path needs an sm_90 device");
    return 0;
  };
  return create_ctx(out, device, CtxKind::Nmfd, plan_nmfd(shape, 1), nullptr, finish);  // loss partials: nmfd_shape_of
}

int nmfb200_nmfd_set_target(nmfb200_ctx* ctx, const void* V, int dtype, void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::Nmfd));
  if (int rc = check_target(V, dtype)) return rc;
  commit_target(ctx, TargetForm::Dense, V, dtype, 0, 0);
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t vin = ctx->d.v_inner();
  int rc = matrix_minmax(V, dtype, (int64_t)ctx->d.B * ctx->d.C, vin, vin, ctx->mm_scratch, ctx->mm_scratch + kMmPartials, st);
  if (rc) return rc;
  if (ctx->tcd) {
    double vsum = 0.0;
    rc = tc_nmfd_set_target(ctx->tcd, V, dtype, &vsum, st);       // synchronises: sum(V) for kappa
    if (rc) return rc;
    tc_nmfd_mark_dirty(ctx->tcd);                         // a new fit: the factors may be anything
    if (ctx->auto_mode)                                   // same conservative rule as the NMF path: heavy-tailed targets stay fp32
      return auto_off_if_heavy_tailed(ctx, vsum, (double)ctx->d.B * ctx->d.C * ctx->d.v_inner(), st);
  }
  return 0;
}

/* ---- batched NMFD / NMF2D / NMF3D: P independent problems of one shape on the fp32 kernels ------------------------ */

namespace {
// The shape of a batch of P NMFD problems (validated): what every problem's launches and counts must fit.
int batched_nmfd_shape_of(int64_t P, int64_t B, int64_t C, int ndim, const int64_t* vdims, int64_t R, const int64_t* kdims,
                          NmfdShape* out) {
  if (P < 1) return fail(NMFB200_ERR_INVALID, "P must be positive");
  NmfdShape d;
  if (int rc = nmfd_shape_of(B, C, ndim, vdims, R, kdims, &d)) return rc;
  // the problems ride on grid z of the sliding kernels (int line index b0 + z) and of wgrad (sliced), on grid x of the
  // column sums, and their loss partials are counted in int
  const int64_t vol = B * C * d.v_inner();
  if (P > INT32_MAX / B)
    return fail(NMFB200_ERR_INVALID, "batched NMFD: P x B must be below 2^31 (the line index of the fp32 kernels)");
  if (nmfd_max_blocks(d) > INT32_MAX / P)
    return fail(NMFB200_ERR_INVALID, "batched NMFD: P x loss partials per problem must be below 2^31");
  const int64_t cs_w = colsum_scratch_floats(C, (int)R, d.w_inner()), cs_h = colsum_scratch_floats(B, (int)R, d.h_inner());
  if ((double)(d.w_inner() > 1 ? cs_w : cs_w / R) * P > (double)kMaxGridX ||
      (double)(d.h_inner() > 1 ? cs_h : cs_h / R) * P > (double)kMaxGridX || ceil_div(R, 64) * P > kMaxGridX)
    return fail(NMFB200_ERR_INVALID, "batched NMFD: P x column-sum blocks must be below 2^31 (grid x of the column sums)");
  if ((double)vol * P > (double)((int64_t)1 << 46)) return fail(NMFB200_ERR_INVALID, "batched NMFD: targets too large");
  *out = d;
  return 0;
}
}  // namespace

int nmfb200_nmfnd_batched_create(nmfb200_ctx** out, int device, int64_t P, int64_t B, int64_t C, int ndim,
                                 const int64_t* vdims, int64_t R, const int64_t* kdims) {
  if (int rc = check_out(out)) return rc;
  NmfdShape d;
  if (int rc = batched_nmfd_shape_of(P, B, C, ndim, vdims, R, kdims, &d)) return rc;
  return create_ctx(out, device, CtxKind::NmfdBatch, plan_nmfd(d, P));
}

int nmfb200_nmfnd_batched_create_ragged(nmfb200_ctx** out, int device, int64_t P, int64_t B, int64_t C, int ndim,
                                        const int64_t* vdims, int64_t R, const int64_t* kdims, const int64_t* lengths) {
  if (int rc = check_out(out)) return rc;
  NmfdShape d;
  if (int rc = batched_nmfd_shape_of(P, B, C, ndim, vdims, R, kdims, &d)) return rc;
  if (!lengths) return fail(NMFB200_ERR_INVALID, "lengths is null");
  if ((double)B * R * P > (double)kMaxGridX)
    return fail(NMFB200_ERR_INVALID, "ragged NMFD batch: P x B x R must be below 2^31 (grid x of the column sums of H)");
  CtxPlan plan;
  if (int rc = plan_nmfd_ragged(d, P, lengths, &plan)) return rc;
  return create_ctx(out, device, CtxKind::NmfdBatch, plan);
}

int nmfb200_nmfd_batched_set_target(nmfb200_ctx* ctx, const void* V, int64_t problem_stride, int dtype, void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::NmfdBatch));
  if (int rc = check_target(V, dtype)) return rc;
  const int64_t vin = ctx->d.v_inner(), rows = (int64_t)ctx->d.B * ctx->d.C;
  if (problem_stride != 0 && problem_stride < rows * vin)
    return fail(NMFB200_ERR_INVALID, "problem stride must be 0 (one shared target) or at least B x C x prod(X)");
  commit_target(ctx, TargetForm::Dense, V, dtype, 0, problem_stride);
  if (ctx->rag)           // a ragged batch: every problem's real positions of each line, even of a shared target
    return matrix_minmax(V, dtype, rows * (vin / ctx->d.L), ctx->d.L, ctx->d.L, ctx->mm_scratch, ctx->mm_scratch + kMmPartials,
                         (cudaStream_t)stream, CellSel{}, ctx->nprob, problem_stride, ctx->rag, true);
  return matrix_minmax(V, dtype, rows, vin, vin, ctx->mm_scratch, ctx->mm_scratch + kMmPartials, (cudaStream_t)stream,
                       CellSel{}, problem_stride ? ctx->nprob : 1, problem_stride);
}

int nmfb200_nmfd_batched_set_active(nmfb200_ctx* ctx, const uint8_t* active, void* stream) {
  (void)stream;
  return set_active(ctx, CtxKind::NmfdBatch, active);
}

int nmfb200_nmfd_plan(int64_t B, int64_t C, int ndim, const int64_t* vdims, int64_t R, const int64_t* kdims, int64_t* out,
                      int n) {
  if (!out || n < NMFB200_NMFD_PLAN_LEN) return fail(NMFB200_ERR_INVALID, "plan buffer too small");
  NmfdShape d;
  if (int rc = nmfd_shape_of(B, C, ndim, vdims, R, kdims, &d)) return rc;
  NmfdPlan p;
  nmfd_plan(d, &p);
  const WgradPlan& w = p.wgrad;
  nmfb200_ctx c;                      // the shape alone, for the ratio stage's views of W and H
  c.kind = CtxKind::Nmfd; c.R = R; c.d = d;
  const int64_t v[NMFB200_NMFD_PLAN_LEN] = {
      p.recon_mt, p.recon_grid.x, p.recon_grid.y, p.recon_grid.z,
      p.dgrad_mt, p.dgrad_nsplit, p.dgrad_grid.x, p.dgrad_grid.y, p.dgrad_grid.z,
      w.mt, w.tp, w.nr, w.no, w.ntt, w.nrg, w.nog, p.wgrad_nsplit,
      apply_update_vec4_shape(factor_view(&c, 0, p.wgrad_nsplit)), apply_update_vec4_shape(factor_view(&c, 1, p.dgrad_nsplit))};
  for (int i = 0; i < NMFB200_NMFD_PLAN_LEN; ++i) out[i] = v[i];
  return 0;
}

int nmfb200_nmfnd_tc_plan(int64_t B, int64_t C, int ndim, const int64_t* vdims, int64_t R, const int64_t* kdims,
                          int64_t* out, int n) {
  if (!out || n < NMFB200_NMFND_TC_PLAN_LEN) return fail(NMFB200_ERR_INVALID, "plan buffer too small");
  NmfdShape d;
  if (int rc = nmfd_shape_of(B, C, ndim, vdims, R, kdims, &d)) return rc;
  TcNmfdPlan p;
  if (const char* why = tc_nmfd_plan(d, &p)) return fail(NMFB200_ERR_INVALID, why);
  const int64_t v[NMFB200_NMFND_TC_PLAN_LEN] = {
      p.prep_w.x, p.prep_w.y, p.prep_w.z, p.prep_h.x, p.prep_h.y, p.prep_h.z, p.recon.x, p.recon.y, p.recon.z,
      p.wgrad.x, p.wgrad.y, p.wgrad.z, p.dgrad.x, p.dgrad.y, p.dgrad.z, p.bslice, p.slices, p.dgrad_rblocks,
      p.loss_blocks, p.ws_w, p.kbs_w, p.ws_h, p.kbs_h, p.hslice, p.hslices, p.Tp, p.padl, p.Lp, p.Lq, p.Cpad, p.nch};
  for (int i = 0; i < NMFB200_NMFND_TC_PLAN_LEN; ++i) out[i] = v[i];
  return 0;
}

int nmfb200_nmf_tc_plan(int64_t N, int64_t C, int64_t R, int precision, int num_sms, int64_t* out, int n) {
  if (!out || n < NMFB200_NMF_TC_PLAN_LEN) return fail(NMFB200_ERR_INVALID, "plan buffer too small");
  if (N < 1 || C < 1 || R < 1) return fail(NMFB200_ERR_INVALID, "N, C, R must be positive");
  if (num_sms < 1) return fail(NMFB200_ERR_INVALID, "num_sms must be positive");
  if (precision != NMFB200_PREC_AUTO && precision != NMFB200_PREC_F16 && precision != NMFB200_PREC_F16_SPLIT)
    return fail(NMFB200_ERR_INVALID, "the tensor-core plan needs precision f16, f16_split or auto");
  if (!tc_shape_supported(N, C, R))
    return fail(NMFB200_ERR_INVALID, "shape not supported by the tensor-core path (need R <= 128)");
  tc_plan(N, C, R, precision == NMFB200_PREC_F16_SPLIT, num_sms, out);
  return 0;
}

/* ---- both kinds: the mask or weights, and the terms of one factor update that every CUDA-core path runs on --- */

namespace {
// set_mask / set_weight: one selector replaces the other
int set_selector(nmfb200_ctx* ctx, CellSel sel, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  TARGET_GUARD(ctx);
  if (is_batch(ctx)) return fail(NMFB200_ERR_INVALID, "batched fits take no mask or weight");
  if (is_sparse(ctx))
    return fail(NMFB200_ERR_INVALID, std::string(sel.kind == kSelWeight ? "a weight" : "a mask") +
                                         " needs a dense target (set_target or nmfd_set_target)");
  cudaStream_t st = (cudaStream_t)stream;
  ctx->sel = sel.p ? sel : CellSel{};
  // the tensor-core paths are bypassed while a selector is set: their operand copies are rebuilt on their next use
  mark_stale(ctx, true, true);
  float* minmax = ctx->mm_scratch + kMmPartials;          // target_minmax: the selected cells only, or all of V again
  if (ctx->kind == CtxKind::Nmf)
    return matrix_minmax(ctx->V, ctx->vdtype, ctx->N, ctx->C, ctx->ldv, ctx->mm_scratch, minmax, st, ctx->sel);
  const int64_t vin = ctx->d.v_inner();
  return matrix_minmax(ctx->V, ctx->vdtype, (int64_t)ctx->d.B * ctx->d.C, vin, vin, ctx->mm_scratch, minmax, st, ctx->sel);
}
}  // namespace

int nmfb200_set_mask(nmfb200_ctx* ctx, const uint8_t* M, void* stream) {
  return set_selector(ctx, CellSel{M, kSelMask}, stream);
}

int nmfb200_set_weight(nmfb200_ctx* ctx, const float* Wt, void* stream) {
  return set_selector(ctx, CellSel{Wt, kSelWeight}, stream);
}

int nmfb200_set_fixed_w(nmfb200_ctx* ctx, const uint8_t* fixed, void* stream) {
  (void)stream;              // nothing is queued: the flags are read by the kernels of later W updates
  CTX_GUARD(ctx, kDenseModels | kinds(CtxKind::PlcaSparse));
  if (is_batch(ctx)) return fail(NMFB200_ERR_INVALID, "batched fits take no fixed components of W");
  if (ctx->kind == CtxKind::PlcaSparse)
    return fail(NMFB200_ERR_INVALID, "sparse PLCA contexts do not update W (its EM step is the caller's)");
  TARGET_GUARD(ctx);
  if (fixed && ctx->ard) return fail(NMFB200_ERR_INVALID, "fixed components of W do not combine with ARD (nmfb200_set_ard)");
  ctx->fixed_w = fixed;
  return 0;
}

namespace {
// The ARD lambda update from W and H (first: the registration's initial lambda, change 0)
int ard_lambda(nmfb200_ctx* c, const float* W, const float* H, bool first, cudaStream_t st) {
  const FactorDims w = factor_dims(c, 0), h = factor_dims(c, 1);
  return ard_update(W, w.rows, w.inner, H, h.rows, h.inner, (int)c->R, c->ard_b, c->ard_c, c->ard_phi, first,
                    c->cs_scratch, c->cs_scratch.n, c->ard_state, st);
}

// What the ARD calls serve: a single NMF or NMFD / NMF2D / NMF3D context (CTX_GUARD) with a target
int ard_check(nmfb200_ctx* ctx) {
  if (is_batch(ctx)) return fail(NMFB200_ERR_INVALID, "batched fits take no ARD");
  TARGET_GUARD(ctx);
  return 0;
}
}  // namespace

int nmfb200_set_ard(nmfb200_ctx* ctx, const float* W, const float* H, double b, double c, double phi, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  if (int rc = ard_check(ctx)) return rc;
  if (!W && !H) { ctx->ard = false; return 0; }
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "set_ard: W and H must both be given (both null clears ARD)");
  auto positive = [](double x) { return std::isfinite(x) && x > 0.0; };
  if (!positive(b) || !positive(c) || !positive(phi)) return fail(NMFB200_ERR_INVALID, "set_ard: b, c and phi must be finite and > 0");
  if (ctx->fixed_w) return fail(NMFB200_ERR_INVALID, "ARD does not combine with fixed components of W (nmfb200_set_fixed_w)");
  NMF_CUDA_CHECK(ctx->ard_state.ensure(ard_state_floats((int)ctx->R)));
  ctx->ard_b = b; ctx->ard_c = c; ctx->ard_phi = phi;
  int rc = ard_lambda(ctx, W, H, true, (cudaStream_t)stream);
  ctx->ard = rc == 0;
  return rc;
}

int nmfb200_ard_update(nmfb200_ctx* ctx, const float* W, const float* H, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  if (int rc = ard_check(ctx)) return rc;
  if (!ctx->ard) return fail(NMFB200_ERR_STATE, "ard_update: ARD is not registered (nmfb200_set_ard)");
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  return ard_lambda(ctx, W, H, false, (cudaStream_t)stream);
}

int nmfb200_ard_read(nmfb200_ctx* ctx, float* lambda, float* pen, float* change, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  if (int rc = ard_check(ctx)) return rc;
  if (!ctx->ard) return fail(NMFB200_ERR_STATE, "ard_read: ARD is not registered (nmfb200_set_ard)");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t R = (size_t)ctx->R;
  const float* state = ctx->ard_state;
  if (lambda) NMF_CUDA_CHECK(cudaMemcpyAsync(lambda, state + 2 * R, R * sizeof(float), cudaMemcpyDefault, st));
  if (pen) NMF_CUDA_CHECK(cudaMemcpyAsync(pen, state + 3 * R, R * sizeof(float), cudaMemcpyDefault, st));
  if (change) NMF_CUDA_CHECK(cudaMemcpyAsync(change, state + 4 * R, sizeof(float), cudaMemcpyDefault, st));
  NMF_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

namespace {
// beta 1 and 2 run on every sparse context; any other beta > 0 only on one set by nmfb200_nmf_set_target_sparse_any_beta,
// every beta on one set by nmfb200_nmf_set_target_observed
int check_sparse_beta(const nmfb200_ctx* ctx, double beta) {
  if (beta == 1.0 || beta == 2.0 || ctx->form == TargetForm::Observed) return 0;
  if (ctx->form != TargetForm::SparseAnyBeta)
    return fail(NMFB200_ERR_INVALID, "sparse targets: beta must be 1 or 2 (densify the target for other beta)");
  if (!(beta > 0.0)) return fail(NMFB200_ERR_INVALID, "sparse targets: beta must be positive");
  return 0;
}

// The terms of one factor's update on the compressed form whose segments are that factor's rows (which = 0: W over CSC,
// 1: H over CSR), all in final form: the numerator (rows x R) into `num`; into `den` the colsum of the other factor (R, beta
// 1), the raw denominator F (other^T other) (rows x R, beta 2) or, at any other beta, the V-free denominator's chunk sum.
// Observed cells: both from one gather at every beta.
int sparse_terms(nmfb200_ctx* ctx, int which, const float* F, const float* other, double beta, float* num, float* den,
                 cudaStream_t st) {
  if (int rc = check_sparse_beta(ctx, beta)) return rc;
  const int R = (int)ctx->R;
  const FactorDims f = factor_dims(ctx, which);
  const int64_t* ptr = which == 0 ? ctx->sp.ccol : ctx->sp.crow;
  const int64_t* idx = which == 0 ? ctx->sp.row : ctx->sp.col;
  const float* val = which == 0 ? ctx->sp.val_t : ctx->sp.val;
  if (ctx->form == TargetForm::Observed)
    return observed_terms(ptr, idx, val, F, other, R, f.rows, beta, num, den, st, which == 0 ? ctx->sp.wt_t : ctx->sp.wt);
  int rc = sparse_numerator(ptr, idx, val, F, other, R, f.rows, beta, num, st);
  if (rc) return rc;
  if (beta != 1.0 && beta != 2.0) {     // the V-free denominator on the dense fp32 plan, its chunks summed as the dense path does
    ApplyArgs chunks = factor_view(ctx, which, ctx->nslab[which]);
    chunks.num = ctx->den;
    rc = simt_nmf_contract_den(F, other, f.rows, f.other_rows, R, beta, chunks.nchunks, ctx->den, ctx->R, chunks.numel, st);
    if (rc) return rc;
    return raw_sum(chunks, den, nullptr, st);
  }
  if (beta == 1.0)                                             // colsum of the OTHER factor, nmf.py:122-131
    return factor_colsum(other, f.other_rows, R, 1, ctx->cs_scratch, ctx->cs_scratch.n, den, st);
  float* G = ctx->sp_gram + (1 - which) * R * R;               // Gram matrix of the other factor
  rc = sparse_gram(other, f.other_rows, R, ctx->sp_gram + 2 * R * R, G, st);
  if (rc) return rc;
  return sparse_rows_times_gram(F, G, f.rows, R, den, st);     // nmf.py:609
}

// CUDA-core contraction of one NMF factor update (which = 0: W, 1: H) into c->num / c->den (chunked partials).
int simt_contract(nmfb200_ctx* c, int which, const float* W, const float* H, double beta, cudaStream_t st) {
  if (beta != 1.0 || c->sel) NMF_CUDA_CHECK(c->den.ensure(c->num.n));
  // W update: F = W (C rows), G = H (N rows), Vm = V^T;  H update: F = H (N rows), G = W (C rows), Vm = V
  const float* fac[2] = {W, H};
  const FactorDims f = factor_dims(c, which);
  return simt_nmf_contract(c->V, c->vdtype, c->ldv, /*trans=*/which == 0, fac[which], fac[1 - which], f.rows, f.other_rows,
                           (int)c->R, beta, c->nslab[which], c->num, c->den, c->R, f.rows * c->R * c->nprob, c->sel, c->C,
                           st, launch_batch(c, which == 0 ? kRagW : kRagH));
}

// The same for NMFD / NMF2D / NMF3D: the ratio tiles Pn (and Pp), then their backward passes (wgrad for W, dgrad for H) into
// c->num and, unless the column sums serve, c->den (split partials).
int nmfd_contract(nmfb200_ctx* c, int which, const float* W, const float* H, double beta, cudaStream_t st) {
  const bool den = !kl_colsum(c, beta);
  if (den) {
    NMF_CUDA_CHECK(c->Pp.ensure(c->Pn.n));
    NMF_CUDA_CHECK(c->den.ensure(c->num.n));
  }
  // a batch: every problem's tiles and split partials in the same launches (slab layout [split][problem][rows][R][inner]; a
  // ragged batch: each problem's own [split][rows][R][inner] at its offset)
  const Batch bt = launch_batch(c, which == 0 ? kRagW : kRagH);
  int rc = nmfd_recon_phi(c->d, c->V, c->vdtype, W, H, beta, c->Pn, c->Pp, nullptr, 0, nullptr, st, c->sel, bt);
  auto grad = [&](const float* P, float* out) {
    return which == 0 ? nmfd_wgrad(c->d, P, H, out, c->nslab[0], st, bt) : nmfd_dgrad(c->d, P, W, out, c->nslab[1], st, bt);
  };
  if (rc == 0) rc = grad(c->Pn, c->num);
  if (rc == 0 && den) rc = grad(c->Pp, c->den);
  return rc;
}

// Both backward passes of one factor (which = 0: W, 1: H) from the current factors, described as the ratio stage's input
// (nmf.py:367-391): partial slabs of numerators and, but for unmasked beta 1, denominators; at unmasked beta 1 the column
// sums of the other factor (nmf.py:122-131) as kl_den; on the NMFD tensor cores the centring term kappa / kappa_vec, with
// `*tc` set.  Terms the kernels leave in final form -- the sparse numerator and denominator, the column sums -- go straight
// to `out` ([numerator | denominator], nmfb200_raw_terms' layout) or, when it is null, to the context's scratch.  Serves
// every path but the NMF tensor-core leaf (tc_update, tc_raw_terms).
int factor_terms(nmfb200_ctx* c, int which, const float* W, const float* H, double beta, float* out, ApplyArgs& a,
                 bool* tc, cudaStream_t st) {
  a = factor_view(c, which, 1);
  const float* fac[2] = {W, H};
  const bool kl = kl_colsum(c, beta);
  // where the final-form terms go without `out`: c->colsum is [colsum(W) | colsum(H)], the sparse raw denominator lives in
  // c->den at beta 2 and on observed cells, and in c->sp_den at other beta (whose c->den holds the chunks)
  if (is_sparse(c) && beta == 2.0 && !out) NMF_CUDA_CHECK(c->den.ensure(c->num.n));
  float* num_out = out ? out : c->num;
  float* den_out = out ? out + a.numel : kl ? c->colsum + (1 - which) * c->R * c->nprob
                 : (beta == 2.0 || c->form == TargetForm::Observed) ? c->den : c->sp_den;
  *tc = c->tcd && use_tc(c, beta);
  if (*tc) {                  // NMFD beta 1: the recon pass also brings both column sums and kappa up to date
    int rc = tc_nmfd_recon(c->tcd, c->V, c->vdtype, W, H, false, nullptr, st);
    if (rc) return rc;
    const float* part; int nsplit;
    rc = which == 0 ? tc_nmfd_wgrad(c->tcd, &part, &nsplit, st) : tc_nmfd_dgrad(c->tcd, &part, &nsplit, st);
    if (rc) return rc;
    const float* cs = tc_nmfd_colsum(c->tcd) + (1 - which) * c->R;
    a.num = part; a.nchunks = nsplit; a.kl_den = cs; a.kappa = tc_nmfd_kappa(c->tcd); a.kappa_vec = cs;
    return 0;
  }
  if (is_sparse(c)) {
    a.num = num_out;
    if (kl) a.kl_den = den_out;
    else a.den = den_out;
    return sparse_terms(c, which, fac[which], fac[1 - which], beta, num_out, den_out, st);
  }
  int rc = is_nmfd(c) ? nmfd_contract(c, which, W, H, beta, st) : simt_contract(c, which, W, H, beta, st);
  if (rc) return rc;
  a.num = c->num; a.nchunks = c->nslab[which];
  if (!kl) { a.den = c->den; return 0; }
  a.kl_den = den_out;
  const FactorDims f = factor_dims(c, which);
  const bool rag_h = c->rag && which == 0;        // a ragged batch's H: each problem's own rows (NMFD: line positions)
  return factor_colsum(fac[1 - which], f.other_rows, (int)c->R, f.other_inner, c->cs_scratch, c->cs_scratch.n, den_out,
                       st, c->nprob, c->active, rag_h ? c->rag.p : nullptr, rag_h ? c->rag_gx[kRagColsum] : 0,
                       rag_h && is_nmfd(c) ? c->d.Lin : 0);
}

// One factor update (which = 0: param = W, 1: param = H) on the kernels that serve this context and beta.  No device guard:
// the entry points select the context's device.
int update_factor(nmfb200_ctx* ctx, int which, float* param, const float* W, const float* H, double beta, double gamma,
                  double l1_reg, double l2_reg, cudaStream_t st) {
  const uint8_t* fixed = which == 0 ? ctx->fixed_w : nullptr;
  const float* pen = ctx->ard ? ctx->ard_state + 3 * ctx->R : nullptr;       // ARD: both factors
  if (ctx->tc && use_tc(ctx, beta))
    return tc_update(ctx->tc, which, param, W, H, beta, gamma, l1_reg, l2_reg, st, fixed, pen);
  ApplyArgs a; bool tc;
  int rc = factor_terms(ctx, which, W, H, beta, nullptr, a, &tc, st);
  if (rc) return rc;
  a.param = param; a.gamma = (float)gamma; a.l1 = (float)l1_reg; a.l2 = (float)l2_reg;
  if (tc) a.absmax_bits = tc_nmfd_begin_update(ctx->tcd, which, st);
  rc = apply_update(a, st, fixed, pen);
  if (rc) return rc;
  if (!tc) mark_stale(ctx, which == 0, which == 1);
  return 0;
}

int sparse_loss_ctx(nmfb200_ctx* ctx, const float* W, const float* H, double beta, double* loss_dev, cudaStream_t st) {
  if (int rc = check_sparse_beta(ctx, beta)) return rc;
  const int R = (int)ctx->R;
  if (ctx->form == TargetForm::Observed)      // every cell's term at the observed cells, nothing elsewhere
    return observed_loss(ctx->sp.crow, ctx->sp.col, ctx->sp.val, H, W, R, ctx->N, beta, ctx->sp_loss_part, loss_dev, st,
                         ctx->sp.wt);
  if (beta != 1.0 && beta != 2.0) {     // pos = sum x^beta over every cell without V, then V_norm - neg at the non-zeros
    int npos = 0;
    int rc = simt_nmf_pow_sum(H, W, ctx->N, ctx->C, R, beta, ctx->loss_blocks, (int)ctx->loss_blocks.n, &npos, st);
    if (rc) return rc;
    return sparse_beta_loss(ctx->sp.crow, ctx->sp.col, ctx->sp.val, H, W, R, ctx->N, beta, ctx->loss_blocks, npos,
                            ctx->sp_loss_part, loss_dev, st);
  }
  const float *pa, *pb;
  int rc;
  if (beta == 1.0) {
    rc = factor_colsum(W, ctx->C, R, 1, ctx->cs_scratch, ctx->cs_scratch.n, ctx->colsum, st);
    if (rc == 0) rc = factor_colsum(H, ctx->N, R, 1, ctx->cs_scratch, ctx->cs_scratch.n, ctx->colsum + R, st);
    pa = ctx->colsum; pb = ctx->colsum + R;
  } else {
    rc = sparse_gram(W, ctx->C, R, ctx->sp_gram + 2 * R * R, ctx->sp_gram, st);
    if (rc == 0) rc = sparse_gram(H, ctx->N, R, ctx->sp_gram + 2 * R * R, ctx->sp_gram + R * R, st);
    pa = ctx->sp_gram; pb = ctx->sp_gram + R * R;
  }
  if (rc) return rc;
  return sparse_loss(ctx->sp.crow, ctx->sp.col, ctx->sp.val, H, W, R, ctx->N, beta, pa, pb,
                     beta == 1.0 ? ctx->sp.vnorm_kl : ctx->sp.vnorm_eu, ctx->sp_loss_part, loss_dev, st);
}
}  // namespace

int nmfb200_target_minmax(nmfb200_ctx* ctx, float* vmin, float* vmax, void* stream) {
  if (!ctx) return fail(NMFB200_ERR_INVALID, "null context");
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return fail(NMFB200_ERR_CUDA, "cannot select the context's device");
  TARGET_GUARD(ctx);
  if (ctx->kind == CtxKind::PlcaSparse) return fail(NMFB200_ERR_INVALID, "wrong context kind");
  float mm[2];
  NMF_CUDA_CHECK(cudaMemcpyAsync(mm, ctx->mm_scratch + kMmPartials, sizeof(mm), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  NMF_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  if (vmin) *vmin = mm[0];
  if (vmax) *vmax = mm[1];
  return 0;
}

int nmfb200_nmf_iterate(nmfb200_ctx* ctx, float* W, float* H, double beta, double gamma, double l1_reg,
                        double l2_reg, int n_iter, void* stream) {
  CTX_GUARD(ctx, kDenseNmf);
  TARGET_GUARD(ctx);
  if (!W || !H || n_iter < 0) return fail(NMFB200_ERR_INVALID, "bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  for (int i = 0; i < n_iter; ++i) {
    int rc = update_factor(ctx, 0, W, W, H, beta, gamma, l1_reg, l2_reg, st);
    if (rc) return rc;
    rc = update_factor(ctx, 1, H, W, H, beta, gamma, l1_reg, l2_reg, st);
    if (rc == 0 && ctx->ard) rc = ard_lambda(ctx, W, H, false, st);
    if (rc) return rc;
  }
  return 0;
}

int nmfb200_nmf_loss_prefetch_w(nmfb200_ctx* ctx, const float* W, const float* H, double beta, double* loss_dev,
                                void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::Nmf));
  TARGET_GUARD(ctx);
  if (!W || !H || !loss_dev) return fail(NMFB200_ERR_INVALID, "null pointer");
  if (!is_sparse(ctx) && use_tc(ctx, beta))
    return tc_loss_prefetch_w(ctx->tc, W, H, beta, loss_dev, (cudaStream_t)stream);
  return nmfb200_loss(ctx, W, H, beta, loss_dev, stream);
}

/* ---- row-sharded W update over peer memory (NVLink, one process per GPU) ---------------------- */

int nmfb200_nmf_peer_supported(const nmfb200_ctx* ctx, double beta) {
  if (!ctx || ctx->kind != CtxKind::Nmf || !has_target(ctx) || ctx->fixed_w || ctx->ard || !use_tc(ctx, beta)) return 0;
  return tc_peer_supported(ctx->tc, beta) ? 1 : 0;
}

int nmfb200_nmf_peer_alloc(nmfb200_ctx* ctx, void* ipc_handle_out) {
  CTX_GUARD(ctx, kinds(CtxKind::Nmf));
  if (!ctx->tc) return fail(NMFB200_ERR_STATE, "the peer-memory W update needs the tensor-core path");
  if (!ipc_handle_out) return fail(NMFB200_ERR_INVALID, "null pointer");
  return tc_peer_alloc(ctx->tc, ipc_handle_out);
}

int nmfb200_nmf_peer_connect(nmfb200_ctx* ctx, int world, int rank, const void* ipc_handles) {
  CTX_GUARD(ctx, kinds(CtxKind::Nmf));
  if (!ctx->tc) return fail(NMFB200_ERR_STATE, "the peer-memory W update needs the tensor-core path");
  if (!ipc_handles) return fail(NMFB200_ERR_INVALID, "null pointer");
  return tc_peer_connect(ctx->tc, world, rank, ipc_handles);
}

int nmfb200_nmf_peer_world(const nmfb200_ctx* ctx) {
  return (ctx && ctx->kind == CtxKind::Nmf && ctx->tc) ? tc_peer_world(ctx->tc) : 0;
}

int nmfb200_nmf_peer_release(nmfb200_ctx* ctx) {
  CTX_GUARD(ctx, kinds(CtxKind::Nmf));
  if (ctx->tc) tc_peer_release(ctx->tc);
  return 0;
}

int nmfb200_nmf_update_w_peer(nmfb200_ctx* ctx, float* W, const float* H, double beta, double gamma, double l1_reg,
                              double l2_reg, void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::Nmf));
  TARGET_GUARD(ctx);
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  if (ctx->ard) return fail(NMFB200_ERR_INVALID, "ARD fits are not sharded (nmfb200_set_ard)");
  if (!nmfb200_nmf_peer_supported(ctx, beta)) return fail(NMFB200_ERR_STATE, "peer-memory W update is not available for this context / beta");
  return tc_update_w_peer(ctx->tc, W, H, beta, gamma, l1_reg, l2_reg, (cudaStream_t)stream);
}

int nmfb200_nmf_contract_only(nmfb200_ctx* ctx, const float* W, const float* H, int which, double beta,
                              void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::Nmf));
  TARGET_GUARD(ctx);
  if (is_sparse(ctx)) return fail(NMFB200_ERR_STATE, "not available for a sparse target");
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (use_tc(ctx, beta)) return tc_contract_only(ctx->tc, W, H, which, beta, st);
  return simt_contract(ctx, which, W, H, beta, st);
}

/* ---- both kinds: the arguments are checked once, then the context's own kernels run ------------------------ */

int nmfb200_sync_factors(nmfb200_ctx* ctx) {
  CTX_GUARD(ctx, kDenseModels);
  // operand copies are rebuilt lazily; the CUDA-core paths read the fp32 factors directly
  mark_stale(ctx, true, true);
  return 0;
}

// update_w / update_h: one factor update (which = 0: param = W, 1: param = H)
static int checked_update(nmfb200_ctx* ctx, int which, float* param, const float* W, const float* H, double beta,
                          double gamma, double l1_reg, double l2_reg, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  TARGET_GUARD(ctx);
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  return update_factor(ctx, which, param, W, H, beta, gamma, l1_reg, l2_reg, (cudaStream_t)stream);
}

int nmfb200_update_w(nmfb200_ctx* ctx, float* W, const float* H, double beta, double gamma, double l1_reg, double l2_reg,
                     void* stream) {
  return checked_update(ctx, 0, W, W, H, beta, gamma, l1_reg, l2_reg, stream);
}

int nmfb200_update_h(nmfb200_ctx* ctx, const float* W, float* H, double beta, double gamma, double l1_reg, double l2_reg,
                     void* stream) {
  return checked_update(ctx, 1, H, W, H, beta, gamma, l1_reg, l2_reg, stream);
}

int nmfb200_loss(nmfb200_ctx* ctx, const float* W, const float* H, double beta, double* loss_dev, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  TARGET_GUARD(ctx);
  if (!W || !H || !loss_dev) return fail(NMFB200_ERR_INVALID, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  // a batch: loss_dev[b] for every active problem b
  if (is_nmfd(ctx)) {
    if (use_tc(ctx, beta)) return tc_nmfd_recon(ctx->tcd, ctx->V, ctx->vdtype, W, H, true, loss_dev, st);
    return nmfd_recon_phi(ctx->d, ctx->V, ctx->vdtype, W, H, beta, nullptr, nullptr, ctx->loss_blocks, (int)ctx->loss_blocks.n,
                          loss_dev, st, ctx->sel, launch_batch(ctx, kRagLoss));
  }
  if (is_sparse(ctx)) return sparse_loss_ctx(ctx, W, H, beta, loss_dev, st);
  if (use_tc(ctx, beta)) return tc_loss(ctx->tc, W, H, beta, loss_dev, st);
  return simt_nmf_loss(ctx->V, ctx->vdtype, ctx->ldv, H, W, ctx->N, ctx->C, (int)ctx->R, beta, ctx->loss_blocks,
                       (int)ctx->loss_blocks.n, loss_dev, ctx->sel, ctx->C, st, launch_batch(ctx, kRagLoss));
}

int64_t nmfb200_raw_terms_numel(const nmfb200_ctx* ctx, int which, double beta) {
  if (!ctx || (which != 0 && which != 1)) return -1;
  const int64_t n = factor_view(ctx, which, 1).numel;
  return kl_colsum(ctx, beta) ? n + ctx->R * ctx->nprob : 2 * n;
}

// The raw terms of one factor's update (which = 0: W, 1: H) into `out`, nmfb200_raw_terms_numel floats: the partial slabs
// summed with the centring term folded in (raw_sum), then the KL column sums at beta 1.
int nmfb200_raw_terms(nmfb200_ctx* ctx, const float* W, const float* H, int which, double beta, float* out, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  TARGET_GUARD(ctx);
  if (!W || !H || !out || (which != 0 && which != 1)) return fail(NMFB200_ERR_INVALID, "bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (ctx->tc && use_tc(ctx, beta) && tc_supports_partial(ctx->tc, beta))
    return tc_raw_terms(ctx->tc, which, W, H, beta, out, st);
  ApplyArgs a; bool tc;
  int rc = factor_terms(ctx, which, W, H, beta, out, a, &tc, st);
  if (rc) return rc;
  float* den_out = out + a.numel;
  if (a.num != out && (rc = raw_sum(a, out, den_out, st))) return rc;        // not already in final form
  if (a.kl_den && a.kl_den != den_out)                  // the NMFD tensor cores keep their column sums
    NMF_CUDA_CHECK(cudaMemcpyAsync(den_out, a.kl_den, (size_t)ctx->R * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (!tc) mark_stale(ctx, false, false);               // no factor changed: NMF's operand copies stay valid
  return 0;
}

// The update's ratio stage on summed raw W terms: one slab, leaving the tensor-core state as update_w does
int nmfb200_w_apply(nmfb200_ctx* ctx, float* W, const float* reduced, double beta, double gamma, double l1_reg,
                    double l2_reg, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  TARGET_GUARD(ctx);
  if (is_batch(ctx)) return fail(NMFB200_ERR_INVALID, "w_apply does not serve batched contexts");
  if (ctx->ard) return fail(NMFB200_ERR_INVALID, "ARD fits are not sharded (nmfb200_set_ard)");
  if (!W || !reduced) return fail(NMFB200_ERR_INVALID, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (ctx->tc && use_tc(ctx, beta)) return tc_w_apply(ctx->tc, W, reduced, beta, gamma, l1_reg, l2_reg, st, ctx->fixed_w);
  ApplyArgs a = factor_view(ctx, 0, 1);     // an NMFD centring term is already folded in by raw_sum
  a.param = W; a.num = reduced; a.gamma = (float)gamma; a.l1 = (float)l1_reg; a.l2 = (float)l2_reg;
  if (kl_colsum(ctx, beta)) a.kl_den = reduced + a.numel;
  else a.den = reduced + a.numel;
  const bool tc = use_tc(ctx, beta);        // here: the NMFD tensor cores
  if (tc) a.absmax_bits = tc_nmfd_begin_update(ctx->tcd, 0, st);
  int rc = apply_update(a, st, ctx->fixed_w);
  if (rc) return rc;
  if (!tc) mark_stale(ctx, true, false);
  return 0;
}

/* ---- masked PLCA: the two gradient terms of one EM step on a partially observed target ---------------------------- */

int nmfb200_plca_masked_terms(nmfb200_ctx* ctx, const float* W, const float* Hz, int which, float* out, double* qobs_dev,
                              void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  if (is_batch(ctx)) return fail(NMFB200_ERR_INVALID, "plca_masked_terms does not serve batched contexts");
  TARGET_GUARD(ctx);
  if (is_sparse(ctx)) return fail(NMFB200_ERR_INVALID, "plca_masked_terms needs a dense target");
  if (ctx->sel.kind == kSelWeight) return fail(NMFB200_ERR_INVALID, "plca_masked_terms takes a mask, not a weight");
  if (!ctx->sel) return fail(NMFB200_ERR_STATE, "plca_masked_terms needs a mask (nmfb200_set_mask)");
  if (ctx->vdtype != NMFB200_DTYPE_F32) return fail(NMFB200_ERR_INVALID, "plca_masked_terms needs an fp32 target");
  if (is_nmfd(ctx) && ctx->R > 256) return fail(NMFB200_ERR_INVALID, "plca_masked_terms: NMFD rank must be <= 256");
  if (!W || !Hz || !out || (which != 0 && which != 1)) return fail(NMFB200_ERR_INVALID, "bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  NMF_CUDA_CHECK(ctx->den.ensure(ctx->num.n));
  const float* V = static_cast<const float*>(ctx->V);
  const uint8_t* M = static_cast<const uint8_t*>(ctx->sel.p);
  int rc;
  if (is_nmfd(ctx)) {        // the fill-mode ratio tiles (and q_O), then their backward passes
    NMF_CUDA_CHECK(ctx->Pp.ensure(ctx->Pn.n));
    rc = nmfd_plca_fill(ctx->d, V, W, Hz, ctx->Pn, ctx->Pp, M, ctx->loss_blocks, (int)ctx->loss_blocks.n, qobs_dev, st);
    auto grad = [&](const float* P, float* part) {
      return which == 0 ? nmfd_wgrad(ctx->d, P, Hz, part, ctx->nslab[0], st)
                        : nmfd_dgrad(ctx->d, P, W, part, ctx->nslab[1], st);
    };
    if (rc == 0) rc = grad(ctx->Pn, ctx->num);
    if (rc == 0) rc = grad(ctx->Pp, ctx->den);
  } else {                   // W: F = W, G = Hz over V^T;  H: F = Hz, G = W over V (simt_contract's roles)
    const FactorDims f = factor_dims(ctx, which);
    const int nch = ctx->nslab[which];
    const int64_t nblocks = simt_plca_fill_blocks(f.rows, nch);
    if (qobs_dev) NMF_CUDA_CHECK(ctx->qobs_part.ensure(nblocks));
    const float* fac[2] = {W, Hz};
    rc = simt_plca_fill_contract(V, ctx->ldv, /*trans=*/which == 0, fac[which], fac[1 - which], f.rows, f.other_rows,
                                 (int)ctx->R, nch, ctx->num, ctx->den, ctx->R, f.rows * ctx->R, M, ctx->C,
                                 qobs_dev ? ctx->qobs_part.p : nullptr, st);
    if (rc == 0 && qobs_dev) rc = sum_partials(ctx->qobs_part, (int)nblocks, qobs_dev, st);
  }
  if (rc) return rc;
  ApplyArgs a = factor_view(ctx, which, ctx->nslab[which]);
  a.num = ctx->num; a.den = ctx->den;
  return raw_sum(a, out, out + a.numel, st);
}

/* ---- coordinate descent at beta 2 (HALS): one sweep per factor update, dense or sparse NMF targets -------------------- */

namespace {
// What the cd calls serve: a single NMF context of rank <= 256 with a dense target and no selector, or a sparse one set by
// set_target_sparse / set_target_sparse_any_beta.
int cd_check(nmfb200_ctx* ctx) {
  if (is_nmfd(ctx)) return fail(NMFB200_ERR_INVALID, "cd: NMFD / NMF2D / NMF3D contexts are not served (NMF only)");
  if (is_batch(ctx)) return fail(NMFB200_ERR_INVALID, "cd: batched contexts are not served");
  if (ctx->R > 256) return fail(NMFB200_ERR_INVALID, "cd: rank must be at most 256");
  TARGET_GUARD(ctx);
  if (ctx->form == TargetForm::Observed) return fail(NMFB200_ERR_INVALID, "cd: observed-cell targets are not served");
  if (ctx->sel) return fail(NMFB200_ERR_INVALID, "cd: contexts with a mask or a weight are not served");
  if (ctx->ard) return fail(NMFB200_ERR_INVALID, "cd: ARD takes the multiplicative updates (nmfb200_set_ard)");
  return 0;
}

// What the batched cd calls serve: a nmfb200_nmf_batched_create context (CTX_GUARD) whose every launch fits grid x.  The
// problems ride on grid x, and the sweep and Gram kernels take more blocks per problem than nmfb200_nmf_batched_create checks.
int cd_batched_check(nmfb200_ctx* ctx) {
  if (ctx->rag) return fail(NMFB200_ERR_INVALID, "batched cd: a ragged batch (nmfb200_nmf_batched_create_ragged) is not served");
  int64_t rpb;
  int nb_n, nb_c;
  sparse_gram_plan(ctx->N, &rpb, &nb_n);
  sparse_gram_plan(ctx->C, &rpb, &nb_c);
  const int64_t per_problem[] = {cd_sweep_blocks(ctx->N > ctx->C ? ctx->N : ctx->C), nb_n > nb_c ? nb_n : nb_c,
                                 ceil_div(ctx->R * ctx->R, 256)};
  for (int64_t blocks : per_problem)
    if (blocks > kMaxGridX / ctx->nprob)
      return fail(NMFB200_ERR_INVALID, "batched cd: B x ceil(max(N, C) / 32) sweep blocks (and B x the Gram blocks) must "
                                       "fit grid x (2^31 - 1)");
  TARGET_GUARD(ctx);
  return 0;
}

// One HALS sweep of W (which = 0) or H (which = 1) in place: A = the beta-2 numerator of that factor's update into c->num
// (dense: the numerator-only contraction's chunk partials; sparse: the gather at the stored entries, in final form), B = the
// other factor's Gram matrix, then the sweep.  A batch runs every active problem in the same four launches, each on its single
// context's plan: A's slabs [chunk][problem][rows][R] (simt_contract's layout), the Grams [2][problem][R^2].
int cd_update_factor(nmfb200_ctx* c, int which, float* W, float* H, double l1_reg, double l2_reg, cudaStream_t st) {
  const int R = (int)c->R;
  const int64_t P = c->nprob;
  const FactorDims f = factor_dims(c, which);
  float* X = which == 0 ? W : H;
  const float* other = which == 0 ? H : W;
  // X / A partials (f, p), the other factor (g) and its Gram (p of the Gram) of problem b
  const Batch bt = launch_batch(c, which == 0 ? kRagW : kRagH);
  int nch = 1;
  int rc;
  if (is_sparse(c)) {         // the compressed form whose segments are X's rows (sparse_terms' choice)
    rc = sparse_numerator(which == 0 ? c->sp.ccol : c->sp.crow, which == 0 ? c->sp.row : c->sp.col,
                          which == 0 ? c->sp.val_t : c->sp.val, X, other, R, f.rows, 2.0, c->num, st);
  } else {
    NMF_CUDA_CHECK(c->sp_gram.ensure(gram_floats(c)));
    nch = c->nslab[which];
    rc = simt_nmf_contract_num(c->V, c->vdtype, c->ldv, /*trans=*/which == 0, other, f.rows, f.other_rows, R, nch, c->num,
                               f.rows * R * P, st, bt);
  }
  if (rc) return rc;
  float* G = c->sp_gram + (1 - which) * P * R * R;
  Batch gbt = bt;
  gbt.f = bt.g; gbt.p = (int64_t)R * R;
  if ((rc = sparse_gram(other, f.other_rows, R, c->sp_gram + 2 * P * R * R, G, st, gbt))) return rc;
  Batch sbt = bt;
  sbt.g = (int64_t)R * R;
  if ((rc = cd_sweep(X, f.rows, R, c->num, nch, f.rows * R * P, G, (float)l1_reg, (float)l2_reg, st, sbt,
                     which == 0 ? c->fixed_w : nullptr)))
    return rc;
  if (!is_sparse(c)) mark_stale(c, which == 0, which == 1);   // the tensor-core operand copies of X are out of date
  return 0;
}

int cd_iterate(nmfb200_ctx* c, float* W, float* H, double l1_reg, double l2_reg, int n_iter, cudaStream_t st) {
  for (int i = 0; i < n_iter; ++i) {
    int rc = cd_update_factor(c, 0, W, H, l1_reg, l2_reg, st);
    if (rc == 0) rc = cd_update_factor(c, 1, W, H, l1_reg, l2_reg, st);
    if (rc) return rc;
  }
  return 0;
}
}  // namespace

int nmfb200_nmf_cd_update(nmfb200_ctx* ctx, float* W, float* H, int which, double l1_reg, double l2_reg, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  if (int rc = cd_check(ctx)) return rc;
  if (!W || !H || (which != 0 && which != 1)) return fail(NMFB200_ERR_INVALID, "bad argument");
  return cd_update_factor(ctx, which, W, H, l1_reg, l2_reg, (cudaStream_t)stream);
}

int nmfb200_nmf_cd_iterate(nmfb200_ctx* ctx, float* W, float* H, double l1_reg, double l2_reg, int n_iter, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  if (int rc = cd_check(ctx)) return rc;
  if (!W || !H || n_iter < 0) return fail(NMFB200_ERR_INVALID, "bad argument");
  return cd_iterate(ctx, W, H, l1_reg, l2_reg, n_iter, (cudaStream_t)stream);
}

int nmfb200_nmf_batched_cd_update(nmfb200_ctx* ctx, float* W, float* H, int which, double l1_reg, double l2_reg,
                                  void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::NmfBatch));
  if (int rc = cd_batched_check(ctx)) return rc;
  if (!W || !H || (which != 0 && which != 1)) return fail(NMFB200_ERR_INVALID, "bad argument");
  return cd_update_factor(ctx, which, W, H, l1_reg, l2_reg, (cudaStream_t)stream);
}

int nmfb200_nmf_batched_cd_iterate(nmfb200_ctx* ctx, float* W, float* H, double l1_reg, double l2_reg, int n_iter,
                                   void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::NmfBatch));
  if (int rc = cd_batched_check(ctx)) return rc;
  if (!W || !H || n_iter < 0) return fail(NMFB200_ERR_INVALID, "bad argument");
  return cd_iterate(ctx, W, H, l1_reg, l2_reg, n_iter, (cudaStream_t)stream);
}

/* ---- coordinate descent at beta 2 on the observed cells of a target (observed_cd.cu) ------------------------------ */

namespace {
// What the observed cd calls serve: a single NMF context whose target was set by set_target_observed / _weighted
// (so R <= 256 and no mask or weight).  nmfb200_nmf_cd_* keeps its own refusal of these contexts.
int observed_cd_check(nmfb200_ctx* ctx) {
  if (is_nmfd(ctx)) return fail(NMFB200_ERR_INVALID, "observed cd: NMFD / NMF2D / NMF3D contexts are not served (NMF only)");
  if (is_batch(ctx)) return fail(NMFB200_ERR_INVALID, "observed cd: batched contexts are not served");
  if (ctx->R > 256) return fail(NMFB200_ERR_INVALID, "observed cd: rank must be at most 256");
  TARGET_GUARD(ctx);
  if (ctx->form != TargetForm::Observed)
    return fail(NMFB200_ERR_INVALID, "observed cd: only targets set by nmfb200_nmf_set_target_observed / _weighted are "
                                     "served (nmfb200_nmf_cd_update serves dense and sparse targets)");
  if (ctx->ard) return fail(NMFB200_ERR_INVALID, "observed cd: ARD takes the multiplicative updates (nmfb200_set_ard)");
  return 0;
}

// One update of W (which = 0, over the CSC form) or H (which = 1, over the CSR form) in place.
int observed_cd_update_factor(nmfb200_ctx* c, int which, float* W, float* H, double l1_reg, double l2_reg,
                              cudaStream_t st) {
  const int R = (int)c->R;
  if (const int64_t nr = observed_cd_workspace_floats(R, c->sp.nnz)) NMF_CUDA_CHECK(c->obs_r.ensure(nr));
  const SparseTarget& s = c->sp;
  if (which == 0)
    return observed_cd(s.ccol, s.row, s.val_t, s.wt_t, W, H, R, c->C, c->obs_r, (float)l1_reg, (float)l2_reg, st,
                       c->fixed_w);
  return observed_cd(s.crow, s.col, s.val, s.wt, H, W, R, c->N, c->obs_r, (float)l1_reg, (float)l2_reg, st);
}
}  // namespace

int nmfb200_nmf_observed_cd_update(nmfb200_ctx* ctx, float* W, float* H, int which, double l1_reg, double l2_reg,
                                   void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  if (int rc = observed_cd_check(ctx)) return rc;
  if (!W || !H || (which != 0 && which != 1)) return fail(NMFB200_ERR_INVALID, "bad argument");
  return observed_cd_update_factor(ctx, which, W, H, l1_reg, l2_reg, (cudaStream_t)stream);
}

int nmfb200_nmf_observed_cd_iterate(nmfb200_ctx* ctx, float* W, float* H, double l1_reg, double l2_reg, int n_iter,
                                    void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  if (int rc = observed_cd_check(ctx)) return rc;
  if (!W || !H || n_iter < 0) return fail(NMFB200_ERR_INVALID, "bad argument");
  for (int i = 0; i < n_iter; ++i) {
    int rc = observed_cd_update_factor(ctx, 0, W, H, l1_reg, l2_reg, (cudaStream_t)stream);
    if (rc == 0) rc = observed_cd_update_factor(ctx, 1, W, H, l1_reg, l2_reg, (cudaStream_t)stream);
    if (rc) return rc;
  }
  return 0;
}

/* ---- batched PLCA: the EM iteration on the raw terms of a batched NMF / NMFD context ---------------------------- */

namespace {
// The floats of plca_iterate's work buffer: [dW | dHz | the EM step's scratch]
struct PlcaWork { int64_t wn, hn, buf; };
PlcaWork plca_work(const nmfb200_ctx* c) {
  const FactorDims w = factor_dims(c, 0);
  return {w.rows * c->R * w.inner * c->nprob, w.other_rows * c->R * w.other_inner * c->nprob,
          plca_em_buf_floats((int)c->R, w.inner, w.other_inner) * c->nprob};
}

// The raw numerator of one factor's update at beta 1 into `out`: the contraction and raw_sum of nmfb200_raw_terms, without
// the column sums PLCA does not use
int plca_numerator(nmfb200_ctx* c, int which, const float* W, const float* Hz, float* out, cudaStream_t st) {
  int rc = is_nmfd(c) ? nmfd_contract(c, which, W, Hz, 1.0, st) : simt_contract(c, which, W, Hz, 1.0, st);
  if (rc) return rc;
  ApplyArgs a = factor_view(c, which, c->nslab[which]);
  a.num = c->num;
  return raw_sum(a, out, nullptr, st);
}
}  // namespace

int64_t nmfb200_plca_work_numel(const nmfb200_ctx* ctx) {
  if (!ctx || !is_batch(ctx)) return -1;
  const PlcaWork w = plca_work(ctx);
  return w.wn + w.hn + w.buf;
}

int nmfb200_plca_iterate(nmfb200_ctx* ctx, float* W, float* H, float* Z, float* Hz, float* work, int flags,
                         const float* W_alpha, const float* H_alpha, const float* Z_alpha, int n_iter, void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  if (!is_batch(ctx)) return fail(NMFB200_ERR_INVALID, "plca_iterate takes a batched NMF or NMFD context");
  if (ctx->rag && is_nmfd(ctx)) return fail(NMFB200_ERR_INVALID, "plca_iterate does not serve a ragged NMFD batch");
  TARGET_GUARD(ctx);
  if (!W || !H || !Z || !Hz || !work || n_iter < 0) return fail(NMFB200_ERR_INVALID, "bad argument");
  if (flags & ~(NMFB200_PLCA_TRAIN_W | NMFB200_PLCA_TRAIN_H | NMFB200_PLCA_TRAIN_Z))
    return fail(NMFB200_ERR_INVALID, "unknown plca_iterate flags");
  if (ctx->R > 256) return fail(NMFB200_ERR_INVALID, "batched PLCA supports rank <= 256");
  cudaStream_t st = (cudaStream_t)stream;
  const PlcaWork pw = plca_work(ctx);
  float* dW = work;
  float* dHz = work + pw.wn;
  float* buf = dHz + pw.hn;
  const FactorDims w = factor_dims(ctx, 0);
  for (int i = 0; i < n_iter; ++i) {
    int rc = plca_numerator(ctx, 0, W, Hz, dW, st);
    if (rc == 0) rc = plca_numerator(ctx, 1, W, Hz, dHz, st);
    if (rc == 0) rc = plca_em(ctx->nprob, w.rows, w.inner, w.other_rows, w.other_inner, (int)ctx->R, W, H, Z, Hz, dW, dHz,
                              W_alpha, H_alpha, Z_alpha, flags, buf, ctx->active, ctx->rag, st);
    if (rc) return rc;
  }
  return 0;
}

int nmfb200_plca_loss(nmfb200_ctx* ctx, const float* W, const float* Hz, const float* norm_dev, double* loss_dev,
                      void* stream) {
  CTX_GUARD(ctx, kDenseModels);
  if (!is_batch(ctx)) return fail(NMFB200_ERR_INVALID, "plca_loss takes a batched NMF or NMFD context");
  if (ctx->rag && is_nmfd(ctx)) return fail(NMFB200_ERR_INVALID, "plca_loss does not serve a ragged NMFD batch");
  TARGET_GUARD(ctx);
  if (!W || !Hz || !norm_dev || !loss_dev) return fail(NMFB200_ERR_INVALID, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  // a ragged batch: problem b's rows, loss chunks and run of partials (loss_part, loss_n) from its plan, as nmfb200_loss
  Batch bt = launch_batch(ctx, kRagLoss);
  bt.scale = norm_dev;
  if (is_nmfd(ctx))
    return nmfd_recon_phi(ctx->d, ctx->V, ctx->vdtype, W, Hz, 1.0, nullptr, nullptr, ctx->loss_blocks, (int)ctx->loss_blocks.n,
                          loss_dev, st, CellSel{}, bt);
  return simt_nmf_loss(ctx->V, ctx->vdtype, ctx->ldv, Hz, W, ctx->N, ctx->C, (int)ctx->R, 1.0, ctx->loss_blocks,
                       (int)ctx->loss_blocks.n, loss_dev, CellSel{}, ctx->C, st, bt);
}

/* ---- sparse-target PLCA: one ratio pass per EM step at the stored entries ------------------------------------------ */

int nmfb200_plca_sparse_create(nmfb200_ctx** out, int device, int64_t N, int64_t C, int64_t R, int64_t nnz) {
  if (int rc = check_out(out)) return rc;
  if (N < 1 || C < 1 || R < 1 || nnz < 0) return fail(NMFB200_ERR_INVALID, "N, C, R must be positive and nnz >= 0");
  if (R > kMaxRank) return fail(NMFB200_ERR_INVALID, kMaxRankMsg);
  if (sparse_gather_blocks(N > C ? N : C) > kMaxGridX)
    return fail(NMFB200_ERR_INVALID, "sparse PLCA: ceil(max(N, C) / 8) gather blocks pass grid x (2^31 - 1)");
  // none of the dense models' workspace: the ratios at the stored entries (at least one float), the loss partials and the
  // two column sums' partials
  auto finish = [&](nmfb200_ctx* c) {
    c->spl_nnz = nnz;
    cudaError_t e = c->spl_P.ensure(std::max(nnz, (int64_t)1));
    if (e == cudaSuccess) e = c->spl_loss_part.ensure(sparse_plca_loss_parts(N));
    if (e == cudaSuccess) e = c->spl_cs_part.ensure(sparse_plca_colsum_parts(C, (int)R) + sparse_plca_colsum_parts(N, (int)R));
    if (e != cudaSuccess) return fail(NMFB200_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
    return 0;
  };
  return create_ctx(out, device, CtxKind::PlcaSparse, CtxPlan{N, C, R}, nullptr, finish);
}

int nmfb200_plca_sparse_set_target(nmfb200_ctx* ctx, const int64_t* crow, const int64_t* col, const float* val,
                                   const int64_t* ccol, const int64_t* row, const int64_t* perm, void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::PlcaSparse));
  (void)stream;
  if (!crow || !ccol || (ctx->spl_nnz > 0 && (!col || !val || !row || !perm)))
    return fail(NMFB200_ERR_INVALID, "bad compressed sparse target");
  SparseTarget sp{crow, col, val, ccol, row};
  sp.perm = perm;
  commit_target(ctx, TargetForm::Sparse, nullptr, NMFB200_DTYPE_F32, 0, 0, sp);
  return 0;
}

int nmfb200_plca_sparse_terms(nmfb200_ctx* ctx, const float* W, const float* Hz, float* out, float norm, double* loss_dev,
                              void* stream) {
  CTX_GUARD(ctx, kinds(CtxKind::PlcaSparse));
  TARGET_GUARD(ctx);
  if (!W || !Hz || (!out && !loss_dev)) return fail(NMFB200_ERR_INVALID, "null pointer");
  float* dW = out;
  float* dHz = out ? out + ctx->C * ctx->R : nullptr;
  const SparseTarget& s = ctx->sp;
  const SparsePlcaTarget t{s.crow, s.col, s.ccol, s.row, s.perm, s.val, ctx->N, ctx->C, (int)ctx->R};
  const SparsePlcaWork ws{ctx->spl_P, ctx->spl_loss_part, ctx->spl_cs_part};
  return sparse_plca_terms(t, ws, W, Hz, dW, dHz, norm, loss_dev, (cudaStream_t)stream);
}

int64_t nmfb200_plca_sparse_device_bytes(const nmfb200_ctx* ctx) {
  if (!ctx || ctx->kind != CtxKind::PlcaSparse) return -1;
  return ctx->spl_P.n * (int64_t)sizeof(float) + (ctx->spl_loss_part.n + ctx->spl_cs_part.n) * (int64_t)sizeof(double);
}

int nmfb200_hoyer_project(int device, float* x, int64_t outer, int64_t D, int64_t inner, const float* k1, const float* k2,
                          void* zeroed_ws, void* stream) {
  if (!x || !k1 || !k2 || !zeroed_ws) return fail(NMFB200_ERR_INVALID, "null pointer");
  if (outer < 1 || inner < 1 || D < 1 || D > 0x7fffffff) return fail(NMFB200_ERR_INVALID, "bad shape");
  DeviceGuard guard(device);
  if (!guard.ok) return fail(NMFB200_ERR_CUDA, "cannot select the device");
  return hoyer_project(x, outer, (int)D, inner, k1, k2, (unsigned char*)zeroed_ws, (cudaStream_t)stream);
}

}  // extern "C"
