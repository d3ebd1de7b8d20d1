// Coordinate descent at beta 2 (HALS, Cichocki & Phan 2009): the sweep stage that takes the place of the ratio stage.
//
// One factor update of  1/2 |V - H W^T|^2 + l1 (sum W + sum H) + l2 / 2 (|W|^2 + |H|^2)  with the other factor fixed: for the
// updated factor X (rows x R), A = the numerator (V^T H for W, V W for H) and B = the other factor's Gram matrix (R x R),
//   for k = 0 .. R-1:  X[c,k] <- max(0, X[c,k] + (A[c,k] - sum_j X[c,j] B[j,k] - l1 - l2 X[c,k]) / (B[k,k] + l2))
// with X[c,j] already updated for j < k.  Every row c is independent; the R column steps of a row are sequential.
//
// One warp owns ROWS rows.  Lane l holds components l, l + 32, ... (RPL of them) of each row's X and A in registers.  B is
// staged through shared memory one panel of 32 columns at a time (every row j of them), so rank 256 needs 33 KB, not 256 KB.
//
// Summation orders (fixed by R alone, whatever the grid or the number of rows; the oracle tolerance rests on them):
//   A[c,k]: 0 + the partial slabs in slab order, each added in fp32 -- raw_sum's order, so A equals nmfb200_raw_terms'
//           numerator at beta 2 bit for bit (one slab: the sparse numerator as it is);
//   sum_j X[c,j] B[j,k]: lane l accumulates j = l, l + 32, l + 64, ... in ascending order with fmaf from 0, then the 32 lane
//           sums are added by an xor butterfly over lane distances 16, 8, 4, 2, 1 (every lane ends with the same bits).
#include "common.cuh"

namespace nmfb200 {

namespace {

constexpr int kPanel = 32;        // columns of B per shared-memory panel: one per lane
constexpr int kPanelLd = 33;      // padded pitch: lane l reads row l + 32 m of a column conflict-free
constexpr int kWarps = 8;
constexpr int kSweepRows = 4;     // rows per warp

// BATCH: bt.n problems, problem b on the single problem's blocks [b nbx, (b + 1) nbx) of grid x, with its X at X + b bt.f,
// its A partials at A + b bt.p within each slab and its B at B + b bt.g; a problem whose bt.active flag is 0 exits at once.
// The single-problem instantiations compile none of it.  FIXED: the columns k with fixed[k] != 0 take no step.
template <int RPL, int ROWS, bool BATCH, bool FIXED = false>
__global__ void __launch_bounds__(256)
cd_sweep_kernel(float* __restrict__ X, int64_t rows, int R, const float* __restrict__ A, int nchunks,
                int64_t chunk_stride, const float* __restrict__ B, float l1, float l2, Batch bt,
                const uint8_t* __restrict__ fixed) {
  __shared__ float Bp[kPanel * RPL * kPanelLd];        // Bp[j][kk] = B[j, 32 m + kk] of panel m, zero outside R x R
  const int lane = threadIdx.x & 31;
  int64_t bx = blockIdx.x;
  if constexpr (BATCH) {
    const int64_t nbx = (rows + kWarps * ROWS - 1) / (kWarps * ROWS);
    const int64_t prob = bx / nbx;
    if (batch_skips(bt.active, prob)) return;
    bx -= prob * nbx;
    X += prob * bt.f; A += prob * bt.p; B += prob * bt.g;
  }
  const int64_t row0 = (bx * kWarps + (threadIdx.x >> 5)) * ROWS;
  float x[ROWS][RPL], a[ROWS][RPL];
#pragma unroll
  for (int q = 0; q < ROWS; ++q) {
    const int64_t row = row0 + q;
#pragma unroll
    for (int m = 0; m < RPL; ++m) {
      const int r = lane + 32 * m;
      const bool in = row < rows && r < R;
      float s = 0.f;
      if (in)
        for (int ch = 0; ch < nchunks; ++ch) s += A[ch * chunk_stride + row * R + r];
      a[q][m] = s;
      x[q][m] = in ? X[row * R + r] : 0.f;
    }
  }

#pragma unroll
  for (int m = 0; m < RPL; ++m) {        // panel m: columns k = 32 m + kk, owned by lane kk's slot m
    __syncthreads();
    for (int i = threadIdx.x; i < kPanel * RPL * kPanel; i += 256) {
      const int j = i / kPanel, kk = i - j * kPanel, k = kPanel * m + kk;
      Bp[j * kPanelLd + kk] = (j < R && k < R) ? B[(int64_t)j * R + k] : 0.f;
    }
    __syncthreads();
    const int kend = min(kPanel, R - kPanel * m);
    for (int kk = 0; kk < kend; ++kk) {
      const float hess = Bp[(kPanel * m + kk) * kPanelLd + kk] + l2;
      float dot[ROWS];
#pragma unroll
      for (int q = 0; q < ROWS; ++q) {
        float p = 0.f;
#pragma unroll
        for (int m2 = 0; m2 < RPL; ++m2) p = fmaf(x[q][m2], Bp[(lane + 32 * m2) * kPanelLd + kk], p);
        dot[q] = p;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int q = 0; q < ROWS; ++q) dot[q] += __shfl_xor_sync(0xffffffffu, dot[q], o);
      // sklearn's `hess != 0` guard: a dead component keeps its column; so does a fixed one
      if (hess != 0.f && lane == kk && !(FIXED && fixed[kPanel * m + kk])) {
#pragma unroll
        for (int q = 0; q < ROWS; ++q) {
          const float v = x[q][m];
          x[q][m] = fmaxf(0.f, v + (a[q][m] - dot[q] - l1 - l2 * v) / hess);
        }
      }
    }
  }

#pragma unroll
  for (int q = 0; q < ROWS; ++q) {
    const int64_t row = row0 + q;
#pragma unroll
    for (int m = 0; m < RPL; ++m) {
      const int r = lane + 32 * m;
      if (row < rows && r < R) X[row * R + r] = x[q][m];
    }
  }
}

}  // namespace

int64_t cd_sweep_blocks(int64_t rows) { return ceil_div(rows, (int64_t)kWarps * kSweepRows); }

int cd_sweep(float* X, int64_t rows, int R, const float* A, int nchunks, int64_t chunk_stride, const float* B, float l1,
             float l2, cudaStream_t st, const Batch& bt, const uint8_t* fixed) {
  if (R < 1 || R > 256) { set_error("cd_sweep: rank must be in [1, 256]"); return 1; }
  if (rows < 1) return 0;
  const int rpl = (R + 31) / 32;
  const int64_t blocks = cd_sweep_blocks(rows);
  if (bt.n < 1 || blocks > kMaxGridX / bt.n) { set_error("cd_sweep: batch x row blocks pass grid x"); return 1; }
  const unsigned gx = (unsigned)(blocks * bt.n);
  const bool batched = bt.n > 1 || bt.active;
  if (fixed && batched) { set_error("cd_sweep: fixed components need a single problem"); return 1; }
#define NMF_CD_B(RPLV, BATCH, FIXED)                                                                                  \
  cd_sweep_kernel<RPLV, kSweepRows, BATCH, FIXED><<<gx, 256, 0, st>>>(X, rows, R, A, nchunks, chunk_stride, B, l1, l2, bt, \
                                                                     fixed)
#define NMF_CD(RPLV)                          \
  do {                                        \
    if (fixed) NMF_CD_B(RPLV, false, true);   \
    else if (batched) NMF_CD_B(RPLV, true, false); \
    else NMF_CD_B(RPLV, false, false);        \
  } while (0)
  if (rpl <= 1) NMF_CD(1);
  else if (rpl <= 2) NMF_CD(2);
  else if (rpl <= 4) NMF_CD(4);
  else NMF_CD(8);
#undef NMF_CD
#undef NMF_CD_B
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace nmfb200
