// The EM step of a batch of PLCA / SIPLCA / SIPLCA2 / SIPLCA3 problems (nmfb200_plca_iterate), after the two raw-terms passes
// of the batched NMF / NMFD contexts.  W and H are viewed as (P, outer, R, inner) -- PLCA: W (P, C, R, 1), H (P, N, R, 1); the
// shift-invariant models flatten their kernel and activation axes into `inner` -- so one kernel serves every model and ndim.
// A ragged batch of PLCA problems (nmfb200_nmf_batched_create_ragged) keeps H, Hz and dHz in the padded (P, N, R) layout and
// runs problem p's H side over its own rag[p].rows rows, as a batch of that many rows does.
#include "../../include/nmf_b200.h"
#include "common.cuh"

namespace nmfb200 {

namespace {

constexpr int kEmThreads = 512;
constexpr int kEmWarps = kEmThreads / 32;

// The factor views, the raw terms and the options of one EM step; per-problem blocks back to back.
struct EmArgs {
  float* W; float* H; float* Z; float* Hz;
  const float* dW; const float* dHz;                     // raw numerators: P contracted with H Z, and with W
  const float* aW; const float* aH; const float* aZ;     // the priors' alphas in the factors' shapes, null: alpha = 1
  float* buf; int64_t buf_floats;                        // scratch per problem (plca_em_buf_floats)
  int64_t wrows, winner, hrows, hinner; int R;
  int flags;                                             // NMFB200_PLCA_TRAIN_W / _H / _Z
  const uint8_t* active;
  const RaggedProblem* rag;                              // a ragged PLCA batch: problem p's H rows are rag[p].rows
};

__device__ __forceinline__ float relu(float x) { return x < 0.f ? 0.f : x; }              // torch.clamp_min(x, 0): NaN stays
__device__ __forceinline__ float thresh(float x) { return x > kEps ? x : kEps; }          // F.threshold(x, eps, eps)

// The rows x R x inner view of one problem's factor, walked in an order fixed by the shape alone: `lanes` = max(1, threads /
// rowlen) row lanes, one column (r, i) per thread so that a warp reads consecutive elements; f(e, r) for element e of
// component r, rows lane, lane + lanes, ... of the thread's columns k = lane rowlen + col; g(k, acc) after each column.
template <class F, class G>
__device__ __forceinline__ void walk(int64_t rows, int R, int64_t inner, F f, G g) {
  const int64_t rowlen = (int64_t)R * inner;
  const int64_t lanes = rowlen >= kEmThreads ? 1 : kEmThreads / rowlen;
  for (int64_t k = threadIdx.x; k < lanes * rowlen; k += kEmThreads) {
    const int64_t lane = k / rowlen, col = k - lane * rowlen;
    const int r = (int)(col / inner);
    float acc = 0.f;
    for (int64_t o = lane; o < rows; o += lanes) acc += f(o * rowlen + col, r);
    g(k, acc);
  }
}

// S[r] = sum over (o, i) of f(o R inner + r inner + i, r): walk's per-column sums go to `buf` (lanes x rowlen floats), then
// warp w sums components w, w + warps, ... over (lane, i) and a shuffle tree.  Ends with the block synchronised.
template <class F>
__device__ void comp_sums(int64_t rows, int R, int64_t inner, F f, float* buf, float* S) {
  walk(rows, R, inner, f, [=](int64_t k, float acc) { buf[k] = acc; });
  __syncthreads();
  const int64_t rowlen = (int64_t)R * inner;
  const int64_t lanes = rowlen >= kEmThreads ? 1 : kEmThreads / rowlen;
  const int warp = threadIdx.x >> 5, l = threadIdx.x & 31;
  for (int r = warp; r < R; r += kEmWarps) {
    float acc = 0.f;
    for (int64_t q = l; q < lanes * inner; q += 32) {
      const int64_t lane = q / inner;
      acc += buf[lane * rowlen + (int64_t)r * inner + (q - lane * inner)];
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (l == 0) S[r] = acc;
  }
  __syncthreads();
}

// f(e, r) for every element of the view, in walk's order
template <class F>
__device__ __forceinline__ void each(int64_t rows, int R, int64_t inner, F f) {
  walk(rows, R, inner, [=](int64_t e, int r) { f(e, r); return 0.f; }, [](int64_t, float) {});
}

// One block per problem (grid x): plca.py's EM step (Z, then W, then H, then Hz = H Z) on that problem's raw terms, every sum
// in comp_sums' order.  A problem whose active flag is 0 returns at once.  RAGGED (a.rag set): every sum over H and every
// write of H and Hz runs over the problem's first rag[p].rows rows, in walk's order for that row count; the padding rows past
// them are neither read nor written.  The problems' blocks stay the padded a.hrows rows apart (hn).
template <bool RAGGED>
__global__ void __launch_bounds__(kEmThreads) plca_em_kernel(EmArgs a) {
  __shared__ float Zold[256], Znew[256], prior[256], S[256];
  __shared__ float zsum;
  const int64_t p = blockIdx.x;
  if (batch_skips(a.active, p)) return;
  const int R = a.R, tid = threadIdx.x;
  const int64_t wn = a.wrows * R * a.winner, hn = a.hrows * R * a.hinner;
  if constexpr (RAGGED) a.hrows = a.rag[p].rows;       // H's rows from here on; hn keeps the padded problem stride
  float* W = a.W + p * wn;
  float* H = a.H + p * hn;
  float* Hz = a.Hz + p * hn;
  float* Z = a.Z + p * R;
  const float* dW = a.dW + p * wn;
  const float* dHz = a.dHz + p * hn;
  const float* aW = a.aW ? a.aW + p * wn : nullptr;
  const float* aH = a.aH ? a.aH + p * hn : nullptr;
  const float* aZ = a.aZ ? a.aZ + p * R : nullptr;
  float* buf = a.buf + p * a.buf_floats;
  const int64_t wi = a.winner, hi = a.hinner;
  for (int r = tid; r < R; r += kEmThreads) { Zold[r] = Z[r]; Znew[r] = Z[r]; }
  __syncthreads();

  bool has_prior = false;
  if (a.flags & NMFB200_PLCA_TRAIN_Z) {                 // plca.py:256-262: Z <- Z relu(sum H dHz); the prior before the alpha
    comp_sums(a.hrows, R, hi, [=](int64_t e, int) { return H[e] * dHz[e]; }, buf, S);
    if (tid < R) {
      float z = Zold[tid] * relu(S[tid]);
      prior[tid] = z;
      if (aZ) z = thresh(z + (aZ[tid] - 1.f));
      Znew[tid] = z;
    }
    __syncthreads();
    if (tid < 32) {
      float acc = 0.f;
      for (int r = tid; r < R; r += 32) acc += Znew[r];
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (tid == 0) zsum = acc;
    }
    __syncthreads();
    if (tid < R) Znew[tid] = Znew[tid] / zsum;
    has_prior = true;
  }

  if (a.flags & NMFB200_PLCA_TRAIN_W) {                 // plca.py:264-275
    if (!has_prior) {                                   // frozen Z: W's column sums are the prior
      comp_sums(a.wrows, R, wi, [=](int64_t e, int) { return W[e] * relu(dW[e]); }, buf, S);
      if (tid < R) prior[tid] = S[tid];
      has_prior = true;
    }
    __syncthreads();
    const float* pr = prior;
    each(a.wrows, R, wi, [=](int64_t e, int r) {
      float t = W[e] * relu(dW[e]);
      t = t / pr[r];
      if (aW) t = thresh(t + (aW[e] - 1.f));
      W[e] = t;
    });
    __syncthreads();
    if (aW) {
      comp_sums(a.wrows, R, wi, [=](int64_t e, int) { return W[e]; }, buf, S);
      const float* sr = S;
      each(a.wrows, R, wi, [=](int64_t e, int r) { W[e] = W[e] / sr[r]; });
    }
  }

  if (a.flags & NMFB200_PLCA_TRAIN_H) {                 // plca.py:277-288, dH = dHz Z with the Z from before the update
    if (!has_prior) {                                   // W and Z frozen: H's own column sums
      const float* zo = Zold;
      comp_sums(a.hrows, R, hi, [=](int64_t e, int r) { return H[e] * relu(dHz[e] * zo[r]); }, buf, S);
      if (tid < R) prior[tid] = S[tid];
    }
    __syncthreads();
    const float *pr = prior, *zo = Zold;
    each(a.hrows, R, hi, [=](int64_t e, int r) {
      float t = H[e] * relu(dHz[e] * zo[r]);
      t = t / pr[r];
      if (aH) t = thresh(t + (aH[e] - 1.f));
      H[e] = t;
    });
    __syncthreads();
    if (aH) {
      comp_sums(a.hrows, R, hi, [=](int64_t e, int) { return H[e]; }, buf, S);
      const float* sr = S;
      each(a.hrows, R, hi, [=](int64_t e, int r) { H[e] = H[e] / sr[r]; });
    }
  }
  __syncthreads();
  const float* zn = Znew;
  each(a.hrows, R, hi, [=](int64_t e, int r) { Hz[e] = H[e] * zn[r]; });           // the next iteration's H Z
  if (a.flags & NMFB200_PLCA_TRAIN_Z)
    for (int r = tid; r < R; r += kEmThreads) Z[r] = Znew[r];
}

}  // namespace

int64_t plca_em_buf_floats(int R, int64_t w_inner, int64_t h_inner) {
  const int64_t rowlen = (int64_t)R * (w_inner > h_inner ? w_inner : h_inner);
  return rowlen > kEmThreads ? rowlen : kEmThreads;
}

int plca_em(int64_t nprob, int64_t wrows, int64_t winner, int64_t hrows, int64_t hinner, int R, float* W, float* H, float* Z,
            float* Hz, const float* dW, const float* dHz, const float* aW, const float* aH, const float* aZ, int flags,
            float* buf, const uint8_t* active, const RaggedProblem* rag, cudaStream_t st) {
  if (R < 1 || R > 256) { set_error("plca_em: rank must be in [1, 256]"); return 1; }
  if (nprob < 1 || nprob > kMaxGridX) { set_error("plca_em: bad problem count"); return 1; }
  const EmArgs a{W, H, Z, Hz, dW, dHz, aW, aH, aZ, buf, plca_em_buf_floats(R, winner, hinner),
                 wrows, winner, hrows, hinner, R, flags, active, rag};
  if (rag) plca_em_kernel<true><<<(unsigned)nprob, kEmThreads, 0, st>>>(a);
  else plca_em_kernel<false><<<(unsigned)nprob, kEmThreads, 0, st>>>(a);
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace nmfb200
