// Relevance update of automatic relevance determination with the l1 prior (Tan and Fevotte, "Automatic relevance
// determination in nonnegative matrix factorization with the beta-divergence", TPAMI 2013): one lambda per component from
// the l1 norms of its columns of W and H.  The sums are the fixed-order column sums of update.cu; one small kernel then
// forms lambda, the penalties of the next ratio stages and the largest relative change.
#include "common.cuh"

namespace nmfb200 {

namespace {

constexpr int kArdThreads = 256;

// One block.  state: [sW R | sH R | lambda R | pen R | change 1].  Thread t walks the components t, t + 256, ...; the block's
// maximum is taken in a fixed tree order (max is exact, so the order only matters for NaN, which fmax drops).
__global__ void __launch_bounds__(kArdThreads)
ard_finish_kernel(float* __restrict__ state, int R, double b, double c, double phi, int first) {
  __shared__ double red[kArdThreads];
  const float* sW = state;
  const float* sH = state + R;
  float* lam = state + 2 * (int64_t)R;
  float* pen = state + 3 * (int64_t)R;
  double mx = 0.0;
  for (int r = threadIdx.x; r < R; r += kArdThreads) {
    const float nl = (float)(((double)sW[r] + (double)sH[r] + b) / c);
    if (!first) {
      const double old = (double)lam[r];
      mx = fmax(mx, fabs((double)nl - old) / old);
    }
    lam[r] = nl;
    pen[r] = (float)(phi / (double)nl);
  }
  red[threadIdx.x] = mx;
  __syncthreads();
  for (int s = kArdThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) state[4 * (int64_t)R] = (float)red[0];
}

}  // namespace

int64_t ard_state_floats(int R) { return 4 * (int64_t)R + 1; }

int ard_update(const float* W, int64_t rows_w, int64_t inner_w, const float* H, int64_t rows_h, int64_t inner_h, int R,
               double b, double c, double phi, bool first, float* scratch, int64_t scratch_floats, float* state,
               cudaStream_t st) {
  if (R < 1) { set_error("ard_update: rank must be positive"); return 1; }
  int rc = factor_colsum(W, rows_w, R, inner_w, scratch, scratch_floats, state, st);
  if (rc == 0) rc = factor_colsum(H, rows_h, R, inner_h, scratch, scratch_floats, state + R, st);
  if (rc) return rc;
  ard_finish_kernel<<<1, kArdThreads, 0, st>>>(state, R, b, c, phi, first ? 1 : 0);
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace nmfb200
