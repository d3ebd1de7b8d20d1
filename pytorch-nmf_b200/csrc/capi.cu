// C ABI of libnmf_b200 (see include/nmf_b200.h): context management and the per-update call graphs.
#include "../../include/nmf_b200.h"

#include <atomic>
#include <new>

#include "common.cuh"
#include "tc_nmf.cuh"
#include "tc_nmfd.cuh"

namespace nmfb200 {
static thread_local std::string g_err;
static std::atomic<int64_t> g_launches{0};
void set_error(const std::string& msg) { g_err = msg; }
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int64_t launch_counter() { return g_launches.load(); }
}  // namespace nmfb200

using namespace nmfb200;

struct nmfb200_ctx {
  int kind = 0;            // 0 = NMF, 1 = NMFD
  int device = 0;
  int precision = NMFB200_PREC_F32;
  bool auto_mode = false;   // precision AUTO: the tensor-core path is used only where it is known to hold the parity bar
  bool tc_off = false;      // AUTO found the target outside the fp16 operand range: fp32 CUDA-core kernels instead
  int64_t N = 0, C = 0, R = 0;
  NmfdShape d{};
  const float* V = nullptr;
  int64_t ldv = 0;
  bool has_target = false;
  // chunked partial numerators / denominators of the CUDA-core path
  float* num = nullptr;
  float* den = nullptr;
  int64_t part_floats = 0;
  int nch_w = 1, nch_h = 1;
  float* colsum = nullptr;        // [2][R]: 0 = colsum(W), 1 = colsum(H)
  float* cs_scratch = nullptr;
  int64_t cs_scratch_floats = 0;
  double* loss_blocks = nullptr;
  int loss_max_blocks = 0;
  float* mm_scratch = nullptr;    // 2048 + 2
  // sparse target (beta 1 / 2): borrowed CSR (rows of V) and CSC (= CSR of V^T) forms, V_norm of nmf.py:161-170
  bool sparse = false;
  const int64_t *sp_crow = nullptr, *sp_col = nullptr, *sp_ccol = nullptr, *sp_row = nullptr;
  const float *sp_val = nullptr, *sp_val_t = nullptr;
  double sp_vnorm_kl = 0.0, sp_vnorm_eu = 0.0;
  float* sp_gram = nullptr;       // [2][R*R] (W^T W, H^T H) + per-block partials
  double* sp_loss_part = nullptr;
  // NMFD
  float* Pn = nullptr;
  float* Pp = nullptr;
  int wgrad_nsplit = 1;
  int dgrad_nsplit = 1;
  // tensor-core path state (tc_nmf.cu / tc_nmfd.cu)
  TcState* tc = nullptr;
  TcNmfdState* tcd = nullptr;
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

#define CTX_GUARD(ctx, want_kind)                                                   \
  if (!(ctx)) return fail(NMFB200_ERR_INVALID, "null context");                     \
  if ((ctx)->kind != (want_kind)) return fail(NMFB200_ERR_INVALID, "wrong context kind"); \
  DeviceGuard _dev_guard((ctx)->device);                                            \
  if (!_dev_guard.ok) return fail(NMFB200_ERR_CUDA, "cannot select the context's device");

int chunks_for(int64_t rows, int64_t cols) {
  int64_t rb = ceil_div(rows, 64), tiles = ceil_div(cols, 64);
  int64_t want = ceil_div(132 * 4, rb);      // a few waves over the 132 SMs of an H100
  if (want > tiles) want = tiles;
  if (want > 32) want = 32;
  if (want < 1) want = 1;
  return (int)want;
}

int ensure_den(nmfb200_ctx* c) {
  if (!c->den) NMF_CUDA_CHECK(cudaMalloc(&c->den, c->part_floats * sizeof(float)));
  return 0;
}

void free_ctx(nmfb200_ctx* c) {
  if (!c) return;
  DeviceGuard guard(c->device);
  if (c->tc) tc_destroy(c->tc);
  if (c->tcd) tc_nmfd_destroy(c->tcd);
  cudaFree(c->num); cudaFree(c->den); cudaFree(c->colsum); cudaFree(c->cs_scratch);
  cudaFree(c->loss_blocks); cudaFree(c->mm_scratch); cudaFree(c->Pn); cudaFree(c->Pp);
  cudaFree(c->sp_gram); cudaFree(c->sp_loss_part);
  delete c;
}

// CUDA-core contraction of one NMF factor update into c->num / c->den (chunked partials).
int simt_contract_w(nmfb200_ctx* c, const float* W, const float* H, double beta, cudaStream_t st) {
  // F = W (C rows), G = H (N rows), Vm = V^T
  if (beta != 1.0) { int e = ensure_den(c); if (e) return e; }
  return simt_nmf_contract(c->V, c->ldv, /*trans=*/1, W, H, c->C, c->N, (int)c->R, beta, c->nch_w, c->num,
                           c->den, c->R, c->C * c->R, st);
}
int simt_contract_h(nmfb200_ctx* c, const float* W, const float* H, double beta, cudaStream_t st) {
  if (beta != 1.0) { int e = ensure_den(c); if (e) return e; }
  return simt_nmf_contract(c->V, c->ldv, /*trans=*/0, H, W, c->N, c->C, (int)c->R, beta, c->nch_h, c->num,
                           c->den, c->R, c->N * c->R, st);
}

bool use_tc(const nmfb200_ctx* c, double beta) {
  return c->tc != nullptr && !c->tc_off && tc_supports_beta(c->tc, beta);
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
  return nmfb200_check_health(stream);
}

int nmfb200_check_health(void* stream) {
  int rc = tc_check_wait_abort((cudaStream_t)stream);
  if (rc == 0) rc = tc_nmfd_check_wait_abort();
  if (rc > 0) return fail(NMFB200_ERR_STATE, "a kernel aborted an internal barrier wait; results are invalid");
  if (rc < 0) return fail(NMFB200_ERR_CUDA, std::string("stream synchronize: ") + cudaGetErrorString(cudaGetLastError()));
  return 0;
}

int nmfb200_nmf_create(nmfb200_ctx** out, int device, int64_t N, int64_t C, int64_t R, int precision) {
  if (!out) return fail(NMFB200_ERR_INVALID, "out is null");
  *out = nullptr;
  if (N < 1 || C < 1 || R < 1) return fail(NMFB200_ERR_INVALID, "N, C, R must be positive");
  if (R > 256) return fail(NMFB200_ERR_INVALID, "rank > 256 is not supported");
  if (precision < NMFB200_PREC_AUTO || precision > NMFB200_PREC_F16_SPLIT)
    return fail(NMFB200_ERR_INVALID, "unknown precision mode");
  DeviceGuard guard(device);
  if (!guard.ok) return fail(NMFB200_ERR_CUDA, "cannot select the requested device");
  nmfb200_ctx* c = new (std::nothrow) nmfb200_ctx();
  if (!c) return fail(NMFB200_ERR_INVALID, "out of host memory");
  c->kind = 0; c->device = device; c->N = N; c->C = C; c->R = R;
  int resolved = precision;
  // AUTO: single-rounded fp16 operands hold the north-star parity (rtol 1e-3) once the ratio tile is kappa-centred;
  // the parity tests check it against the reference at the configuration shapes
  if (precision == NMFB200_PREC_AUTO) resolved = tc_shape_supported(N, C, R) ? NMFB200_PREC_F16 : NMFB200_PREC_F32;
  if (resolved != NMFB200_PREC_F32 && !tc_shape_supported(N, C, R)) {
    delete c;
    return fail(NMFB200_ERR_INVALID, "shape not supported by the tensor-core path (need R <= 128)");
  }
  c->precision = resolved;
  c->auto_mode = precision == NMFB200_PREC_AUTO;
  c->nch_w = chunks_for(C, N);
  c->nch_h = chunks_for(N, C);
  int64_t pf = (int64_t)c->nch_w * C * R;
  if ((int64_t)c->nch_h * N * R > pf) pf = (int64_t)c->nch_h * N * R;
  c->part_floats = pf;
  int64_t csf = colsum_scratch_floats(N > C ? N : C, (int)R, 1);
  c->cs_scratch_floats = csf;
  c->loss_max_blocks = simt_nmf_max_blocks(N, C);
  cudaError_t e = cudaSuccess;
  if (e == cudaSuccess) e = cudaMalloc(&c->num, pf * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&c->colsum, 2 * R * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&c->cs_scratch, csf * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&c->loss_blocks, (size_t)c->loss_max_blocks * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&c->mm_scratch, 2050 * sizeof(float));
  if (e != cudaSuccess) {
    free_ctx(c);
    return fail(NMFB200_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
  }
  if (resolved != NMFB200_PREC_F32) {
    int rc = tc_create(&c->tc, device, N, C, R, resolved == NMFB200_PREC_F16_SPLIT);
    if (rc) { free_ctx(c); return rc; }
  }
  *out = c;
  return 0;
}

void nmfb200_destroy(nmfb200_ctx* ctx) { free_ctx(ctx); }

int nmfb200_precision(const nmfb200_ctx* ctx) {
  if (!ctx) return -100;
  return ctx->tc_off ? NMFB200_PREC_F32 : ctx->precision;
}

int nmfb200_precision_for_beta(const nmfb200_ctx* ctx, double beta) {
  if (!ctx) return -100;
  if (ctx->kind == 1) return (ctx->tcd && !ctx->tc_off && tc_nmfd_supported(ctx->d, beta)) ? NMFB200_PREC_F16 : NMFB200_PREC_F32;
  if (ctx->kind != 0 || !use_tc(ctx, beta)) return NMFB200_PREC_F32;
  // beta != 1 kernels read only the hi halves of the operand copies
  return (beta == 1.0 || beta == 2.0) ? ctx->precision : NMFB200_PREC_F16;
}

int nmfb200_nmf_plan(int64_t N, int64_t C, int64_t R, int64_t* out, int n) {
  if (!out || n < NMFB200_NMF_PLAN_LEN) return fail(NMFB200_ERR_INVALID, "plan buffer too small");
  if (N < 1 || C < 1 || R < 1) return fail(NMFB200_ERR_INVALID, "N, C, R must be positive");
  if (R > 256) return fail(NMFB200_ERR_INVALID, "rank > 256 is not supported");
  const int nch_w = chunks_for(C, N), nch_h = chunks_for(N, C);
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
  if (R > 256) return fail(NMFB200_ERR_INVALID, "rank > 256 is not supported");
  int64_t rpb_n, rpb_c;
  int nb_n, nb_c;
  sparse_gram_plan(N, &rpb_n, &nb_n);               // H^T H: the W update's beta-2 denominator, the beta-2 loss
  sparse_gram_plan(C, &rpb_c, &nb_c);               // W^T W: the H update's, the loss
  const int64_t v[NMFB200_SPARSE_PLAN_LEN] = {sparse_rpl((int)R), sparse_gram_passes((int)R), rpb_n, nb_n, rpb_c, nb_c,
                                              sparse_gather_blocks(N), sparse_gather_blocks(C)};
  for (int i = 0; i < NMFB200_SPARSE_PLAN_LEN; ++i) out[i] = v[i];
  return 0;
}

int nmfb200_nmf_set_target(nmfb200_ctx* ctx, const float* V, int64_t ldv, void* stream) {
  CTX_GUARD(ctx, 0);
  if (!V || ldv < ctx->C) return fail(NMFB200_ERR_INVALID, "bad target pointer / leading dimension");
  cudaStream_t st = (cudaStream_t)stream;
  ctx->V = V; ctx->ldv = ldv; ctx->has_target = true; ctx->sparse = false;
  int rc = matrix_minmax(V, ctx->N, ctx->C, ldv, ctx->mm_scratch, ctx->mm_scratch + 2048, st);
  if (rc) return rc;
  ctx->tc_off = false;
  if (ctx->tc) {
    rc = tc_set_target(ctx->tc, V, ldv, ctx->mm_scratch + 2048, st);
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
      // ... and for heavy-tailed targets (max / mean > 64: spectrogram-like, lognormal, ...).  Measured on the lognormal
      // fixtures of tests/golden/reference_r2.npz (30 iterations, tolerance rtol 1e-3): f16 34x, f16_split 2x, f32 0.1x of
      // the tolerance -- MU on such targets converges slowly and keeps the per-update operand rounding instead of
      // averaging it out as it does on well-conditioned data (uniform-like targets: 0.17x after 200 iterations).
      if (!ctx->tc_off) {
        double vsum = 0.0;
        float mm[2] = {0.f, 0.f};
        rc = tc_target_sum(ctx->tc, &vsum, st);
        if (rc) return rc;
        NMF_CUDA_CHECK(cudaMemcpyAsync(mm, ctx->mm_scratch + 2048, sizeof(mm), cudaMemcpyDeviceToHost, st));
        NMF_CUDA_CHECK(cudaStreamSynchronize(st));
        const double mean = vsum / ((double)ctx->N * (double)ctx->C);
        ctx->tc_off = !(mean > 0.0) || (double)mm[1] > 64.0 * mean;
      }
    }
  }
  return 0;
}

/* ---- sparse targets (beta 1 and 2): nmf.py:603-638 without the dense product ------------------------------ */

int nmfb200_nmf_set_target_sparse(nmfb200_ctx* ctx, int64_t nnz, const int64_t* crow, const int64_t* col, const float* val,
                                  const int64_t* ccol, const int64_t* row, const float* val_t, double v_norm_kl,
                                  double v_norm_eu, void* stream) {
  CTX_GUARD(ctx, 0);
  (void)stream;
  if (nnz < 0 || !crow || !ccol || (nnz > 0 && (!col || !val || !row || !val_t)))
    return fail(NMFB200_ERR_INVALID, "bad compressed sparse target");
  if (!ctx->sp_gram) {
    const int64_t R = ctx->R;
    NMF_CUDA_CHECK(cudaMalloc(&ctx->sp_gram, (size_t)(2 * R * R + sparse_gram_part_floats((int)R)) * sizeof(float)));
    NMF_CUDA_CHECK(cudaMalloc(&ctx->sp_loss_part, (size_t)sparse_gather_blocks(ctx->N) * sizeof(double)));
  }
  ctx->sp_crow = crow; ctx->sp_col = col; ctx->sp_val = val; ctx->sp_ccol = ccol; ctx->sp_row = row; ctx->sp_val_t = val_t;
  ctx->sp_vnorm_kl = v_norm_kl; ctx->sp_vnorm_eu = v_norm_eu;
  ctx->sparse = true; ctx->has_target = true; ctx->V = nullptr; ctx->tc_off = true;      // the dense kernels are out of play
  return 0;
}

namespace {
// Raw terms of one factor's update on the compressed form whose segments are that factor's rows (which = 0: W over CSC,
// 1: H over CSR): the numerator (rows x R) into `num`; into `den` the colsum of the other factor (R, beta 1) or the raw
// denominator F (other^T other) (rows x R, beta 2).  Shared by the update and nmfb200_nmf_raw_terms.
int sparse_terms(nmfb200_ctx* ctx, int which, const float* F, const float* other, double beta, float* num, float* den,
                 cudaStream_t st) {
  if (beta != 1.0 && beta != 2.0) return fail(NMFB200_ERR_INVALID, "sparse targets: beta must be 1 or 2 (densify the target for other beta)");
  const int R = (int)ctx->R;
  const int64_t rows = which == 0 ? ctx->C : ctx->N, orows = which == 0 ? ctx->N : ctx->C;
  const int64_t* ptr = which == 0 ? ctx->sp_ccol : ctx->sp_crow;
  const int64_t* idx = which == 0 ? ctx->sp_row : ctx->sp_col;
  const float* val = which == 0 ? ctx->sp_val_t : ctx->sp_val;
  int rc = sparse_numerator(ptr, idx, val, F, other, R, rows, beta, num, st);
  if (rc) return rc;
  if (beta == 1.0)                                             // colsum of the OTHER factor, nmf.py:122-131
    return factor_colsum(other, orows, R, 1, ctx->cs_scratch, ctx->cs_scratch_floats, den, st);
  float* G = ctx->sp_gram + (1 - which) * R * R;               // Gram matrix of the other factor
  rc = sparse_gram(other, orows, R, ctx->sp_gram + 2 * R * R, G, st);
  if (rc) return rc;
  return sparse_rows_times_gram(F, G, rows, R, den, st);       // nmf.py:609
}

// one factor update: sparse_terms into the context's scratch, then the ratio stage
int sparse_update(nmfb200_ctx* ctx, int which, float* F, const float* other, double beta, double gamma, double l1_reg,
                  double l2_reg, cudaStream_t st) {
  const int R = (int)ctx->R;
  const int64_t rows = which == 0 ? ctx->C : ctx->N;
  if (beta == 2.0) {
    int rc = ensure_den(ctx);
    if (rc) return rc;
  }
  float* den = beta == 1.0 ? ctx->colsum + (1 - which) * R : ctx->den;
  int rc = sparse_terms(ctx, which, F, other, beta, ctx->num, den, st);
  if (rc) return rc;
  ApplyArgs a{};
  a.param = F; a.numel = rows * R; a.R = R; a.inner = 1; a.rowlen = R;
  a.num = ctx->num; a.den = beta == 1.0 ? nullptr : den; a.nchunks = 1; a.chunk_stride = 0;
  a.ldp = R; a.kl_den = beta == 1.0 ? den : nullptr; a.out_scale = nullptr;
  a.gamma = (float)gamma; a.l1 = (float)l1_reg; a.l2 = (float)l2_reg; a.absmax_bits = nullptr;
  return apply_update(a, st);
}

int sparse_loss_ctx(nmfb200_ctx* ctx, const float* W, const float* H, double beta, double* loss_dev, cudaStream_t st) {
  if (beta != 1.0 && beta != 2.0) return fail(NMFB200_ERR_INVALID, "sparse targets: beta must be 1 or 2");
  const int R = (int)ctx->R;
  const float *pa, *pb;
  int rc;
  if (beta == 1.0) {
    rc = factor_colsum(W, ctx->C, R, 1, ctx->cs_scratch, ctx->cs_scratch_floats, ctx->colsum, st);
    if (rc == 0) rc = factor_colsum(H, ctx->N, R, 1, ctx->cs_scratch, ctx->cs_scratch_floats, ctx->colsum + R, st);
    pa = ctx->colsum; pb = ctx->colsum + R;
  } else {
    rc = sparse_gram(W, ctx->C, R, ctx->sp_gram + 2 * R * R, ctx->sp_gram, st);
    if (rc == 0) rc = sparse_gram(H, ctx->N, R, ctx->sp_gram + 2 * R * R, ctx->sp_gram + R * R, st);
    pa = ctx->sp_gram; pb = ctx->sp_gram + R * R;
  }
  if (rc) return rc;
  return sparse_loss(ctx->sp_crow, ctx->sp_col, ctx->sp_val, H, W, R, ctx->N, beta, pa, pb,
                     beta == 1.0 ? ctx->sp_vnorm_kl : ctx->sp_vnorm_eu, ctx->sp_loss_part, loss_dev, st);
}
}  // namespace

int nmfb200_target_minmax(nmfb200_ctx* ctx, float* vmin, float* vmax, void* stream) {
  if (!ctx) return fail(NMFB200_ERR_INVALID, "null context");
  DeviceGuard guard(ctx->device);
  if (!guard.ok) return fail(NMFB200_ERR_CUDA, "cannot select the context's device");
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  float mm[2];
  NMF_CUDA_CHECK(cudaMemcpyAsync(mm, ctx->mm_scratch + 2048, sizeof(mm), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  NMF_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  if (vmin) *vmin = mm[0];
  if (vmax) *vmax = mm[1];
  return 0;
}

int nmfb200_nmf_sync_factors(nmfb200_ctx* ctx, const float* W, const float* H, void* stream) {
  CTX_GUARD(ctx, 0);
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  if (ctx->tc) tc_mark_dirty(ctx->tc, true, true);
  return 0;   // operand copies are rebuilt lazily; the CUDA-core path reads the fp32 factors directly
}

int nmfb200_nmf_update_w(nmfb200_ctx* ctx, float* W, const float* H, double beta, double gamma, double l1_reg,
                         double l2_reg, void* stream) {
  CTX_GUARD(ctx, 0);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (ctx->sparse) return sparse_update(ctx, 0, W, H, beta, gamma, l1_reg, l2_reg, st);
  if (use_tc(ctx, beta)) return tc_update_w(ctx->tc, W, H, beta, gamma, l1_reg, l2_reg, st);
  int rc = simt_contract_w(ctx, W, H, beta, st);
  if (rc) return rc;
  float* kl = nullptr;
  if (beta == 1.0) {
    kl = ctx->colsum + ctx->R;
    rc = factor_colsum(H, ctx->N, (int)ctx->R, 1, ctx->cs_scratch, ctx->cs_scratch_floats, kl, st);
    if (rc) return rc;
  }
  ApplyArgs a{};
  a.param = W; a.numel = ctx->C * ctx->R; a.R = (int)ctx->R; a.inner = 1; a.rowlen = ctx->R;
  a.num = ctx->num; a.den = beta == 1.0 ? nullptr : ctx->den; a.nchunks = ctx->nch_w;
  a.chunk_stride = ctx->C * ctx->R; a.ldp = ctx->R; a.kl_den = kl; a.out_scale = nullptr;
  a.gamma = (float)gamma; a.l1 = (float)l1_reg; a.l2 = (float)l2_reg; a.absmax_bits = nullptr;
  rc = apply_update(a, st);
  if (rc) return rc;
  if (ctx->tc) tc_mark_dirty(ctx->tc, true, false);
  return 0;
}

int nmfb200_nmf_update_h(nmfb200_ctx* ctx, const float* W, float* H, double beta, double gamma, double l1_reg,
                         double l2_reg, void* stream) {
  CTX_GUARD(ctx, 0);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (ctx->sparse) return sparse_update(ctx, 1, H, W, beta, gamma, l1_reg, l2_reg, st);
  if (use_tc(ctx, beta)) return tc_update_h(ctx->tc, W, H, beta, gamma, l1_reg, l2_reg, st);
  int rc = simt_contract_h(ctx, W, H, beta, st);
  if (rc) return rc;
  float* kl = nullptr;
  if (beta == 1.0) {
    kl = ctx->colsum;
    rc = factor_colsum(W, ctx->C, (int)ctx->R, 1, ctx->cs_scratch, ctx->cs_scratch_floats, kl, st);
    if (rc) return rc;
  }
  ApplyArgs a{};
  a.param = H; a.numel = ctx->N * ctx->R; a.R = (int)ctx->R; a.inner = 1; a.rowlen = ctx->R;
  a.num = ctx->num; a.den = beta == 1.0 ? nullptr : ctx->den; a.nchunks = ctx->nch_h;
  a.chunk_stride = ctx->N * ctx->R; a.ldp = ctx->R; a.kl_den = kl; a.out_scale = nullptr;
  a.gamma = (float)gamma; a.l1 = (float)l1_reg; a.l2 = (float)l2_reg; a.absmax_bits = nullptr;
  rc = apply_update(a, st);
  if (rc) return rc;
  if (ctx->tc) tc_mark_dirty(ctx->tc, false, true);
  return 0;
}

int nmfb200_nmf_iterate(nmfb200_ctx* ctx, float* W, float* H, double beta, double gamma, double l1_reg,
                        double l2_reg, int n_iter, void* stream) {
  CTX_GUARD(ctx, 0);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H || n_iter < 0) return fail(NMFB200_ERR_INVALID, "bad argument");
  if (use_tc(ctx, beta)) return tc_iterate(ctx->tc, W, H, beta, gamma, l1_reg, l2_reg, n_iter, (cudaStream_t)stream);
  for (int i = 0; i < n_iter; ++i) {
    int rc = nmfb200_nmf_update_w(ctx, W, H, beta, gamma, l1_reg, l2_reg, stream);
    if (rc) return rc;
    rc = nmfb200_nmf_update_h(ctx, W, H, beta, gamma, l1_reg, l2_reg, stream);
    if (rc) return rc;
  }
  return 0;
}

int nmfb200_nmf_loss(nmfb200_ctx* ctx, const float* W, const float* H, double beta, double* loss_dev,
                     void* stream) {
  CTX_GUARD(ctx, 0);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H || !loss_dev) return fail(NMFB200_ERR_INVALID, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (ctx->sparse) return sparse_loss_ctx(ctx, W, H, beta, loss_dev, st);
  if (use_tc(ctx, beta) && tc_supports_loss(ctx->tc, beta)) return tc_loss(ctx->tc, W, H, beta, loss_dev, st);
  return simt_nmf_loss(ctx->V, ctx->ldv, H, W, ctx->N, ctx->C, (int)ctx->R, beta, ctx->loss_blocks,
                       ctx->loss_max_blocks, loss_dev, st);
}

int nmfb200_nmf_loss_prefetch_w(nmfb200_ctx* ctx, const float* W, const float* H, double beta, double* loss_dev,
                                void* stream) {
  CTX_GUARD(ctx, 0);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H || !loss_dev) return fail(NMFB200_ERR_INVALID, "null pointer");
  if (!ctx->sparse && use_tc(ctx, beta) && tc_supports_loss(ctx->tc, beta))
    return tc_loss_prefetch_w(ctx->tc, W, H, beta, loss_dev, (cudaStream_t)stream);
  return nmfb200_nmf_loss(ctx, W, H, beta, loss_dev, stream);
}

int64_t nmfb200_nmf_w_partial_numel(const nmfb200_ctx* ctx, double beta) {
  if (!ctx || ctx->kind != 0) return -1;
  return beta == 1.0 ? ctx->C * ctx->R + ctx->R : 2 * ctx->C * ctx->R;
}

int nmfb200_nmf_w_partial(nmfb200_ctx* ctx, const float* W, const float* H, double beta, float* partial,
                          void* stream) {
  CTX_GUARD(ctx, 0);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (ctx->sparse) return fail(NMFB200_ERR_STATE, "not available for a sparse target");
  if (!W || !H || !partial) return fail(NMFB200_ERR_INVALID, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (use_tc(ctx, beta) && tc_supports_partial(ctx->tc, beta)) return tc_w_partial(ctx->tc, W, H, beta, partial, st);
  int rc = simt_contract_w(ctx, W, H, beta, st);
  if (rc) return rc;
  const int64_t CR = ctx->C * ctx->R;
  rc = reduce_chunks(ctx->num, ctx->nch_w, CR, ctx->C, (int)ctx->R, ctx->R, partial, st);
  if (rc) return rc;
  if (beta == 1.0)
    return factor_colsum(H, ctx->N, (int)ctx->R, 1, ctx->cs_scratch, ctx->cs_scratch_floats, partial + CR, st);
  return reduce_chunks(ctx->den, ctx->nch_w, CR, ctx->C, (int)ctx->R, ctx->R, partial + CR, st);
}

int64_t nmfb200_nmf_raw_terms_numel(const nmfb200_ctx* ctx, int which, double beta) {
  if (!ctx || ctx->kind != 0 || (which != 0 && which != 1)) return -1;
  const int64_t rows = which == 0 ? ctx->C : ctx->N;
  return beta == 1.0 ? rows * ctx->R + ctx->R : 2 * rows * ctx->R;
}

int nmfb200_nmf_raw_terms(nmfb200_ctx* ctx, const float* W, const float* H, int which, double beta, float* out,
                          void* stream) {
  CTX_GUARD(ctx, 0);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H || !out || (which != 0 && which != 1)) return fail(NMFB200_ERR_INVALID, "bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t rows = which == 0 ? ctx->C : ctx->N;
  const int64_t RR = rows * ctx->R;
  if (ctx->sparse) return sparse_terms(ctx, which, which == 0 ? W : H, which == 0 ? H : W, beta, out, out + RR, st);
  if (use_tc(ctx, beta) && tc_supports_partial(ctx->tc, beta)) return tc_raw_terms(ctx->tc, which, W, H, beta, out, st);
  int rc = which == 0 ? simt_contract_w(ctx, W, H, beta, st) : simt_contract_h(ctx, W, H, beta, st);
  if (rc) return rc;
  const int nch = which == 0 ? ctx->nch_w : ctx->nch_h;
  rc = reduce_chunks(ctx->num, nch, RR, rows, (int)ctx->R, ctx->R, out, st);
  if (rc) return rc;
  if (beta == 1.0) {      // nmf.py:122-131: the KL denominator is the column sum of the OTHER factor
    const float* other = which == 0 ? H : W;
    return factor_colsum(other, which == 0 ? ctx->N : ctx->C, (int)ctx->R, 1, ctx->cs_scratch, ctx->cs_scratch_floats,
                         out + RR, st);
  }
  return reduce_chunks(ctx->den, nch, RR, rows, (int)ctx->R, ctx->R, out + RR, st);
}

/* ---- row-sharded W update over peer memory (NVLink, one process per GPU) ---------------------- */

int nmfb200_nmf_peer_supported(const nmfb200_ctx* ctx, double beta) {
  if (!ctx || ctx->kind != 0 || !ctx->tc || ctx->tc_off || !ctx->has_target) return 0;
  return (tc_supports_beta(ctx->tc, beta) && tc_peer_supported(ctx->tc, beta)) ? 1 : 0;
}

int nmfb200_nmf_peer_alloc(nmfb200_ctx* ctx, void* ipc_handle_out) {
  CTX_GUARD(ctx, 0);
  if (!ctx->tc) return fail(NMFB200_ERR_STATE, "the peer-memory W update needs the tensor-core path");
  if (!ipc_handle_out) return fail(NMFB200_ERR_INVALID, "null pointer");
  return tc_peer_alloc(ctx->tc, ipc_handle_out);
}

int nmfb200_nmf_peer_connect(nmfb200_ctx* ctx, int world, int rank, const void* ipc_handles) {
  CTX_GUARD(ctx, 0);
  if (!ctx->tc) return fail(NMFB200_ERR_STATE, "the peer-memory W update needs the tensor-core path");
  if (!ipc_handles) return fail(NMFB200_ERR_INVALID, "null pointer");
  return tc_peer_connect(ctx->tc, world, rank, ipc_handles);
}

int nmfb200_nmf_peer_world(const nmfb200_ctx* ctx) {
  return (ctx && ctx->kind == 0 && ctx->tc) ? tc_peer_world(ctx->tc) : 0;
}

int nmfb200_nmf_peer_release(nmfb200_ctx* ctx) {
  CTX_GUARD(ctx, 0);
  if (ctx->tc) tc_peer_release(ctx->tc);
  return 0;
}

int nmfb200_nmf_update_w_peer(nmfb200_ctx* ctx, float* W, const float* H, double beta, double gamma, double l1_reg,
                              double l2_reg, void* stream) {
  CTX_GUARD(ctx, 0);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  if (!nmfb200_nmf_peer_supported(ctx, beta)) return fail(NMFB200_ERR_STATE, "peer-memory W update is not available for this context / beta");
  return tc_update_w_peer(ctx->tc, W, H, beta, gamma, l1_reg, l2_reg, (cudaStream_t)stream);
}

int nmfb200_nmf_w_apply(nmfb200_ctx* ctx, float* W, const float* reduced, double beta, double gamma,
                        double l1_reg, double l2_reg, void* stream) {
  CTX_GUARD(ctx, 0);
  if (!W || !reduced) return fail(NMFB200_ERR_INVALID, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (use_tc(ctx, beta)) return tc_w_apply(ctx->tc, W, reduced, beta, gamma, l1_reg, l2_reg, st);
  const int64_t CR = ctx->C * ctx->R;
  ApplyArgs a{};
  a.param = W; a.numel = CR; a.R = (int)ctx->R; a.inner = 1; a.rowlen = ctx->R;
  a.num = reduced; a.den = beta == 1.0 ? nullptr : reduced + CR; a.nchunks = 1; a.chunk_stride = 0;
  a.ldp = ctx->R; a.kl_den = beta == 1.0 ? reduced + CR : nullptr; a.out_scale = nullptr;
  a.gamma = (float)gamma; a.l1 = (float)l1_reg; a.l2 = (float)l2_reg; a.absmax_bits = nullptr;
  int rc = apply_update(a, st);
  if (rc) return rc;
  if (ctx->tc) tc_mark_dirty(ctx->tc, true, false);
  return 0;
}

int nmfb200_nmf_contract_only(nmfb200_ctx* ctx, const float* W, const float* H, int which, double beta,
                              void* stream) {
  CTX_GUARD(ctx, 0);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (ctx->sparse) return fail(NMFB200_ERR_STATE, "not available for a sparse target");
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (use_tc(ctx, beta)) return tc_contract_only(ctx->tc, W, H, which, beta, st);
  return which == 0 ? simt_contract_w(ctx, W, H, beta, st) : simt_contract_h(ctx, W, H, beta, st);
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
  *d = NmfdShape{(int)B, (int)C, (int)L, (int)R, (int)T, (int)(L - T + 1)};
  d->X1 = (int)X[0]; d->X2 = (int)X[1]; d->T1 = (int)K[0]; d->T2 = (int)K[1];
  return 0;
}

// The ratio stage's view of one NMFD factor (which = 0: W, 1: H): rows of R components x `inner` elements, one partial slab
// per split.
static ApplyArgs nmfd_apply_shape(const NmfdShape& d, int which, int nsplit) {
  const int64_t inner = which == 0 ? d.w_inner() : d.h_inner();
  ApplyArgs a{};
  a.numel = (int64_t)(which == 0 ? d.C : d.B) * d.R * inner; a.R = d.R; a.inner = inner; a.rowlen = (int64_t)d.R * inner;
  a.chunk_stride = a.numel; a.ldp = a.rowlen; a.nchunks = nsplit; a.out_scale = nullptr; a.absmax_bits = nullptr;
  return a;
}

static int nmfd_create_impl(nmfb200_ctx** out, int device, int64_t B, int64_t C, int ndim, const int64_t* vdims,
                            int64_t R, const int64_t* kdims, int precision) {
  if (!out) return fail(NMFB200_ERR_INVALID, "out is null");
  *out = nullptr;
  NmfdShape shape;
  if (int rc = nmfd_shape_of(B, C, ndim, vdims, R, kdims, &shape)) return rc;
  if (precision != NMFB200_PREC_AUTO && precision != NMFB200_PREC_F32 && precision != NMFB200_PREC_F16)
    return fail(NMFB200_ERR_INVALID, "NMFD precision must be auto, f32 or f16");
  const bool one_d = shape.one_d();
  if (!one_d && precision == NMFB200_PREC_F16)
    return fail(NMFB200_ERR_INVALID, "NMF2D / NMF3D run on the fp32 kernels (precision auto or f32)");
  DeviceGuard guard(device);
  if (!guard.ok) return fail(NMFB200_ERR_CUDA, "cannot select the requested device");
  nmfb200_ctx* c = new (std::nothrow) nmfb200_ctx();
  if (!c) return fail(NMFB200_ERR_INVALID, "out of host memory");
  c->kind = 1; c->device = device; c->precision = precision == NMFB200_PREC_F32 ? NMFB200_PREC_F32 : NMFB200_PREC_F16; c->R = R;
  c->auto_mode = precision == NMFB200_PREC_AUTO;
  c->d = shape;
  c->dgrad_nsplit = nmfd_dgrad_nsplit(c->d);
  c->wgrad_nsplit = nmfd_wgrad_nsplit(c->d);
  int64_t pf = (int64_t)c->wgrad_nsplit * C * R * c->d.w_inner();
  int64_t hf = (int64_t)c->dgrad_nsplit * B * R * c->d.h_inner();
  if (hf > pf) pf = hf;
  c->part_floats = pf;
  int64_t cs1 = colsum_scratch_floats(C, (int)R, c->d.w_inner()), cs2 = colsum_scratch_floats(B, (int)R, c->d.h_inner());
  c->cs_scratch_floats = cs1 > cs2 ? cs1 : cs2;
  c->loss_max_blocks = nmfd_max_blocks(c->d);
  cudaError_t e = cudaSuccess;
  if (e == cudaSuccess) e = cudaMalloc(&c->num, pf * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&c->colsum, 2 * R * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&c->cs_scratch, c->cs_scratch_floats * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&c->loss_blocks, (size_t)c->loss_max_blocks * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&c->mm_scratch, 2050 * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&c->Pn, (size_t)B * C * c->d.v_inner() * sizeof(float));
  if (e != cudaSuccess) {
    free_ctx(c);
    return fail(NMFB200_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e));
  }
  if (c->precision != NMFB200_PREC_F32 && one_d) {       // the tensor-core kernels cover the one-axis case
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess && prop.major == 9) {
      int rc = tc_nmfd_create(&c->tcd, c->d);          // beta = 1 runs as wgmma sliding GEMMs (tc_nmfd.cu)
      if (rc) { free_ctx(c); return rc; }
    } else if (precision == NMFB200_PREC_F16) {
      free_ctx(c);
      return fail(NMFB200_ERR_INVALID, "the tensor-core NMFD path needs an sm_90 device");
    }
  }
  *out = c;
  return 0;
}

int nmfb200_nmfd_create(nmfb200_ctx** out, int device, int64_t B, int64_t C, int64_t L, int64_t R, int64_t T,
                        int precision) {
  return nmfd_create_impl(out, device, B, C, 1, &L, R, &T, precision);
}

int nmfb200_nmfnd_create(nmfb200_ctx** out, int device, int64_t B, int64_t C, int ndim, const int64_t* vdims,
                         int64_t R, const int64_t* kdims, int precision) {
  return nmfd_create_impl(out, device, B, C, ndim, vdims, R, kdims, precision);
}

int nmfb200_nmfd_set_target(nmfb200_ctx* ctx, const float* V, void* stream) {
  CTX_GUARD(ctx, 1);
  if (!V) return fail(NMFB200_ERR_INVALID, "null target");
  ctx->V = V; ctx->has_target = true;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t vin = ctx->d.v_inner();
  int rc = matrix_minmax(V, (int64_t)ctx->d.B * ctx->d.C, vin, vin, ctx->mm_scratch, ctx->mm_scratch + 2048, st);
  if (rc) return rc;
  ctx->tc_off = false;
  if (ctx->tcd) {
    double vsum = 0.0;
    rc = tc_nmfd_set_target(ctx->tcd, V, &vsum, st);       // synchronises: sum(V) for kappa
    if (rc) return rc;
    tc_nmfd_mark_dirty(ctx->tcd);                         // a new fit: the factors may be anything
    if (ctx->auto_mode) {                                 // same conservative rule as the NMF path: heavy-tailed targets stay fp32
      float mm[2] = {0.f, 0.f};
      NMF_CUDA_CHECK(cudaMemcpyAsync(mm, ctx->mm_scratch + 2048, sizeof(mm), cudaMemcpyDeviceToHost, st));
      NMF_CUDA_CHECK(cudaStreamSynchronize(st));
      const double mean = vsum / ((double)ctx->d.B * ctx->d.C * ctx->d.L);
      ctx->tc_off = !(mean > 0.0) || (double)mm[1] > 64.0 * mean;
    }
  }
  return 0;
}

// beta = 1 on tensor cores: both column-sum vectors (KL denominators, nmf.py:122-131, and kappa), then the recon pass
static bool nmfd_use_tc(const nmfb200_ctx* c, double beta) {
  return c->tcd != nullptr && !c->tc_off && tc_nmfd_supported(c->d, beta);
}
static int nmfd_tc_recon(nmfb200_ctx* c, const float* W, const float* H, bool loss, double* loss_dev, cudaStream_t st) {
  return tc_nmfd_recon(c->tcd, c->V, W, H, loss, loss_dev, st);
}

static int nmfd_phi(nmfb200_ctx* c, const float* W, const float* H, double beta, cudaStream_t st) {
  if (beta != 1.0) {
    if (!c->Pp) NMF_CUDA_CHECK(cudaMalloc(&c->Pp, (size_t)c->d.B * c->d.C * c->d.v_inner() * sizeof(float)));
    int e = ensure_den(c);
    if (e) return e;
  }
  return nmfd_recon_phi(c->d, c->V, W, H, beta, c->Pn, c->Pp, nullptr, 0, nullptr, st);
}

// Both backward passes of one factor (which = 0: W, 1: H) from the current factors, described as the ratio stage's input:
// split partial numerators (+ denominators for beta != 1), the KL column sums, the centring term of the tensor-core path.
// Shared by the update (nmf.py:367-391) and by nmfb200_nmfd_raw_terms.  `tc` reports which path produced the terms.
static int nmfd_terms(nmfb200_ctx* ctx, const float* W, const float* H, int which, double beta, ApplyArgs& a, bool* tc,
                      cudaStream_t st) {
  const NmfdShape& d = ctx->d;
  a = nmfd_apply_shape(d, which, 1);
  *tc = nmfd_use_tc(ctx, beta);
  if (*tc) {
    int rc = nmfd_tc_recon(ctx, W, H, false, nullptr, st);
    if (rc) return rc;
    const float* part; int nsplit;
    rc = which == 0 ? tc_nmfd_wgrad(ctx->tcd, &part, &nsplit, st) : tc_nmfd_dgrad(ctx->tcd, &part, &nsplit, st);
    if (rc) return rc;
    a.num = part; a.den = nullptr; a.nchunks = nsplit;
    const float* cs = tc_nmfd_colsum(ctx->tcd) + (which == 0 ? d.R : 0);       // [colsum_W | colsum_H]
    a.kl_den = cs; a.kappa = tc_nmfd_kappa(ctx->tcd); a.kappa_vec = cs;
    return 0;
  }
  if (ctx->tcd) tc_nmfd_mark_dirty(ctx->tcd);            // this pass bypasses the tensor-core state
  int rc = nmfd_phi(ctx, W, H, beta, st);
  if (rc) return rc;
  const int nsplit = which == 0 ? ctx->wgrad_nsplit : ctx->dgrad_nsplit;
  rc = which == 0 ? nmfd_wgrad(d, ctx->Pn, H, ctx->num, nsplit, st) : nmfd_dgrad(d, ctx->Pn, W, ctx->num, nsplit, st);
  if (rc) return rc;
  float* kl = nullptr;
  if (beta == 1.0) {                                     // nmf.py:122-131: column sums of the OTHER factor
    kl = ctx->colsum + (which == 0 ? d.R : 0);
    rc = which == 0 ? factor_colsum(H, d.B, d.R, d.h_inner(), ctx->cs_scratch, ctx->cs_scratch_floats, kl, st)
                    : factor_colsum(W, d.C, d.R, d.w_inner(), ctx->cs_scratch, ctx->cs_scratch_floats, kl, st);
  } else {
    rc = which == 0 ? nmfd_wgrad(d, ctx->Pp, H, ctx->den, nsplit, st) : nmfd_dgrad(d, ctx->Pp, W, ctx->den, nsplit, st);
  }
  if (rc) return rc;
  a.num = ctx->num; a.den = beta == 1.0 ? nullptr : ctx->den; a.nchunks = nsplit; a.kl_den = kl;
  return 0;
}

int nmfb200_nmfd_plan(int64_t B, int64_t C, int ndim, const int64_t* vdims, int64_t R, const int64_t* kdims, int64_t* out,
                      int n) {
  if (!out || n < NMFB200_NMFD_PLAN_LEN) return fail(NMFB200_ERR_INVALID, "plan buffer too small");
  NmfdShape d;
  if (int rc = nmfd_shape_of(B, C, ndim, vdims, R, kdims, &d)) return rc;
  NmfdPlan p;
  nmfd_plan(d, &p);
  const WgradPlan& w = p.wgrad;
  const int64_t v[NMFB200_NMFD_PLAN_LEN] = {
      p.recon_mt, p.recon_grid.x, p.recon_grid.y, p.recon_grid.z,
      p.dgrad_mt, p.dgrad_nsplit, p.dgrad_grid.x, p.dgrad_grid.y, p.dgrad_grid.z,
      w.mt, w.tp, w.nr, w.no, w.ntt, w.nrg, w.nog, p.wgrad_nsplit,
      apply_update_vec4_shape(nmfd_apply_shape(d, 0, p.wgrad_nsplit)), apply_update_vec4_shape(nmfd_apply_shape(d, 1, p.dgrad_nsplit))};
  for (int i = 0; i < NMFB200_NMFD_PLAN_LEN; ++i) out[i] = v[i];
  return 0;
}

static int nmfd_update(nmfb200_ctx* ctx, const float* W, const float* H, int which, float* param, double beta, double gamma,
                       double l1_reg, double l2_reg, cudaStream_t st) {
  ApplyArgs a; bool tc;
  int rc = nmfd_terms(ctx, W, H, which, beta, a, &tc, st);
  if (rc) return rc;
  a.param = param; a.gamma = (float)gamma; a.l1 = (float)l1_reg; a.l2 = (float)l2_reg;
  if (tc) a.absmax_bits = tc_nmfd_begin_update(ctx->tcd, which, st);
  return apply_update(a, st);
}

int nmfb200_nmfd_update_w(nmfb200_ctx* ctx, float* W, const float* H, double beta, double gamma, double l1_reg,
                          double l2_reg, void* stream) {
  CTX_GUARD(ctx, 1);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  return nmfd_update(ctx, W, H, 0, W, beta, gamma, l1_reg, l2_reg, (cudaStream_t)stream);
}

int nmfb200_nmfd_update_h(nmfb200_ctx* ctx, const float* W, float* H, double beta, double gamma, double l1_reg,
                          double l2_reg, void* stream) {
  CTX_GUARD(ctx, 1);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H) return fail(NMFB200_ERR_INVALID, "null factor pointer");
  return nmfd_update(ctx, W, H, 1, H, beta, gamma, l1_reg, l2_reg, (cudaStream_t)stream);
}

int nmfb200_nmfd_sync_factors(nmfb200_ctx* ctx) {
  CTX_GUARD(ctx, 1);
  if (ctx->tcd) tc_nmfd_mark_dirty(ctx->tcd);
  return 0;
}

int64_t nmfb200_nmfd_raw_terms_numel(const nmfb200_ctx* ctx, int which, double beta) {
  if (!ctx || ctx->kind != 1 || (which != 0 && which != 1)) return -1;
  const NmfdShape& d = ctx->d;
  const int64_t n = (int64_t)(which == 0 ? d.C : d.B) * d.R * (which == 0 ? d.w_inner() : d.h_inner());
  return beta == 1.0 ? n + d.R : 2 * n;
}

int nmfb200_nmfd_raw_terms(nmfb200_ctx* ctx, const float* W, const float* H, int which, double beta, float* out,
                           void* stream) {
  CTX_GUARD(ctx, 1);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H || !out || (which != 0 && which != 1)) return fail(NMFB200_ERR_INVALID, "bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  ApplyArgs a; bool tc;
  int rc = nmfd_terms(ctx, W, H, which, beta, a, &tc, st);
  if (rc) return rc;
  rc = raw_sum(a, out, a.den ? out + a.numel : nullptr, st);
  if (rc) return rc;
  if (beta == 1.0)
    NMF_CUDA_CHECK(cudaMemcpyAsync(out + a.numel, a.kl_den, (size_t)ctx->d.R * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}

int nmfb200_nmfd_loss(nmfb200_ctx* ctx, const float* W, const float* H, double beta, double* loss_dev,
                      void* stream) {
  CTX_GUARD(ctx, 1);
  if (!ctx->has_target) return fail(NMFB200_ERR_STATE, "set_target has not been called");
  if (!W || !H || !loss_dev) return fail(NMFB200_ERR_INVALID, "null pointer");
  if (nmfd_use_tc(ctx, beta)) return nmfd_tc_recon(ctx, W, H, true, loss_dev, (cudaStream_t)stream);
  return nmfd_recon_phi(ctx->d, ctx->V, W, H, beta, nullptr, nullptr, ctx->loss_blocks, ctx->loss_max_blocks,
                        loss_dev, (cudaStream_t)stream);
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
