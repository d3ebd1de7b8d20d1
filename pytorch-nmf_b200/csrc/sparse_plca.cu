// Sparse-target PLCA (PLSA on a count matrix): the two gradients of one EM step (plca.py:252-253) at the stored entries of V
// only, from ONE ratio per entry at the current factors W (C x R) and Hz = H diag(Z) (N x R):
//
//   P[n,c] = vn / (hz_n . w_c + eps)            at each stored entry (vn = V / sum V)
//   dHz[n,:] = sum_{c in row n} P[n,c] W[c,:]   dW[c,:] = sum_{n in col c} P[n,c] Hz[n,:]
//
// Pass 1 walks the CSR rows, one warp per row: the warp keeps hz_n in registers, gathers w_c of each entry, forms the dot
// product and P once, accumulates dHz and writes P to an nnz-long buffer.  Pass 2 walks the CSC columns, one warp per column,
// reading P through the CSR position of each entry (perm) and accumulating dW: no dot product.  Each lane owns the rank slots
// lane + 32 k and the dot product is reduced by the xor shuffle of sparse_nmf.cu's gathers, so at R <= 256 x, P, dHz and dW are
// bit for bit those gathers' beta-1 numerators (sparse_numerator) on the factor pair (W, Hz).  Above rank 256 pass 1 takes the
// dot product over 256-wide rank blocks and writes P only; both numerators then come from the P gather, one rank block of 256
// per grid y.
//
// Loss (metrics.kl_div of norm q against the de-normalised target, plca.py:245), x = norm (hz_n . w_c), t = vn norm:
//   sum_nnz [t (log(t + eps) - log(x + eps)) - t] + norm sum_r colsum(W)[r] colsum(Hz)[r]
// A cell that stores nothing contributes its x only.  The per-entry terms ride on pass 1 (one double partial per block), the
// column sums are double partials over row blocks, and one block sums both in a fixed order.  No atomics anywhere: every sum
// runs in an order fixed by the sparsity pattern and R.
#include "common.cuh"

namespace nmfb200 {

namespace {

constexpr int kRankBlock = 256;
constexpr int kColsumMaxBlocks = 1024;

// the per-entry loss term of pass 1 (v: the normalised value, dot: the model's cell)
__device__ __forceinline__ double plca_entry_loss(float v, float dot, float norm) {
  const float t = v * norm, x = norm * dot;
  return (double)t * ((double)logf(t + kEps) - (double)logf(x + kEps)) - (double)t;
}

// per-block sum of the warps' loss terms (every lane of a warp holds the same value), in warp order
__device__ __forceinline__ void plca_block_loss(double lacc, double* loss_part) {
  __shared__ double sh[8];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = lacc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < 8; ++k) t += sh[k];
    loss_part[blockIdx.x] = t;
  }
}

// Pass 1 at R <= 256: one warp per CSR row; dHz (null: the loss alone) and P; LOSS: one loss partial per block
template <int RPL, bool LOSS>
__global__ void __launch_bounds__(256)
plca_rows_kernel(const int64_t* __restrict__ crow, const int64_t* __restrict__ col, const float* __restrict__ val,
                 const float* __restrict__ Hz, const float* __restrict__ W, int R, int64_t N, float* __restrict__ P,
                 float* __restrict__ dHz, float norm, double* __restrict__ loss_part) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  double lacc = 0.0;
  if (row < N) {
    float hs[RPL], acc[RPL];
#pragma unroll
    for (int k = 0; k < RPL; ++k) {
      const int r = lane + 32 * k;
      hs[k] = r < R ? Hz[row * R + r] : 0.f;
      acc[k] = 0.f;
    }
    const int64_t e0 = crow[row], e1 = crow[row + 1];
    for (int64_t e = e0; e < e1; ++e) {
      const int64_t c = col[e];
      const float v = val[e];
      float w[RPL];
#pragma unroll
      for (int k = 0; k < RPL; ++k) {
        const int r = lane + 32 * k;
        w[k] = r < R ? W[c * R + r] : 0.f;
      }
      float dot = 0.f;
#pragma unroll
      for (int k = 0; k < RPL; ++k) dot = fmaf(w[k], hs[k], dot);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
      const float p = v / (dot + kEps);                                  // plca.py:252
#pragma unroll
      for (int k = 0; k < RPL; ++k) acc[k] = fmaf(p, w[k], acc[k]);
      if (lane == 0) P[e] = p;
      if (LOSS) lacc += plca_entry_loss(v, dot, norm);
    }
    if (dHz) {
#pragma unroll
      for (int k = 0; k < RPL; ++k) {
        const int r = lane + 32 * k;
        if (r < R) dHz[row * R + r] = acc[k];
      }
    }
  }
  if (LOSS) plca_block_loss(lacc, loss_part);
}

// Pass 1 above rank 256: the dot product over rank blocks of 256 (8 slots per lane each), then P; no numerator
template <bool LOSS>
__global__ void __launch_bounds__(256)
plca_rows_blocked_kernel(const int64_t* __restrict__ crow, const int64_t* __restrict__ col, const float* __restrict__ val,
                         const float* __restrict__ Hz, const float* __restrict__ W, int R, int64_t N, float* __restrict__ P,
                         float norm, double* __restrict__ loss_part) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  double lacc = 0.0;
  if (row < N) {
    const float* hz = Hz + row * R;
    const int64_t e0 = crow[row], e1 = crow[row + 1];
    for (int64_t e = e0; e < e1; ++e) {
      const float* w = W + col[e] * R;
      float dot = 0.f;
      for (int r0 = 0; r0 < R; r0 += kRankBlock) {
#pragma unroll
        for (int k = 0; k < kRankBlock / 32; ++k) {
          const int r = r0 + lane + 32 * k;
          if (r < R) dot = fmaf(w[r], hz[r], dot);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
      const float v = val[e];
      if (lane == 0) P[e] = v / (dot + kEps);
      if (LOSS) lacc += plca_entry_loss(v, dot, norm);
    }
  }
  if (LOSS) plca_block_loss(lacc, loss_part);
}

// out[seg, rank block y] = sum_{e in segment seg} P[perm[e]] F[idx[e], :] (perm null: P[e]), one warp per segment, the rank
// slots y 256 + lane + 32 k
template <int RPL>
__global__ void __launch_bounds__(256)
plca_gather_kernel(const int64_t* __restrict__ ptr, const int64_t* __restrict__ idx, const int64_t* __restrict__ perm,
                   const float* __restrict__ P, const float* __restrict__ F, int R, int64_t nseg, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t seg = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (seg >= nseg) return;
  const int rb = blockIdx.y * kRankBlock;
  float acc[RPL];
#pragma unroll
  for (int k = 0; k < RPL; ++k) acc[k] = 0.f;
  const int64_t e0 = ptr[seg], e1 = ptr[seg + 1];
  for (int64_t e = e0; e < e1; ++e) {
    const int64_t j = idx[e];
    const float p = P[perm ? perm[e] : e];
#pragma unroll
    for (int k = 0; k < RPL; ++k) {
      const int r = rb + lane + 32 * k;
      acc[k] = fmaf(p, r < R ? F[j * R + r] : 0.f, acc[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < RPL; ++k) {
    const int r = rb + lane + 32 * k;
    if (r < R) out[seg * R + r] = acc[k];
  }
}

// part[b, r] = sum over the rows [b rpb, min(rows, (b + 1) rpb)) of F[row, r], in double, in row order
__global__ void __launch_bounds__(256)
plca_colsum_part_kernel(const float* __restrict__ F, int64_t rows, int R, int64_t rpb, double* __restrict__ part) {
  const int r = blockIdx.y * 256 + threadIdx.x;
  if (r >= R) return;
  const int64_t r0 = (int64_t)blockIdx.x * rpb, r1 = min(rows, r0 + rpb);
  double s = 0.0;
  for (int64_t i = r0; i < r1; ++i) s += (double)F[i * R + r];
  part[(int64_t)blockIdx.x * R + r] = s;
}

// *out = sum(loss_part) + norm sum_r (sum_b wpart[b, r]) (sum_b hpart[b, r]): one block, strided per thread, then a fixed tree
__global__ void __launch_bounds__(256)
plca_loss_final_kernel(const double* __restrict__ loss_part, int64_t nparts, const double* __restrict__ wpart, int nbw,
                       const double* __restrict__ hpart, int nbh, int R, double norm, double* __restrict__ out) {
  __shared__ double sa[256], sb[256];
  double a = 0.0, b = 0.0;
  for (int64_t i = threadIdx.x; i < nparts; i += 256) a += loss_part[i];
  for (int r = threadIdx.x; r < R; r += 256) {
    double cw = 0.0, ch = 0.0;
    for (int k = 0; k < nbw; ++k) cw += wpart[(int64_t)k * R + r];
    for (int k = 0; k < nbh; ++k) ch += hpart[(int64_t)k * R + r];
    b += cw * ch;
  }
  sa[threadIdx.x] = a;
  sb[threadIdx.x] = b;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { sa[threadIdx.x] += sa[threadIdx.x + o]; sb[threadIdx.x] += sb[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sa[0] + norm * sb[0];
}

int launch_rows(const SparsePlcaTarget& t, const float* W, const float* Hz, float* P, float* dHz, float norm,
                double* loss_part, cudaStream_t st) {
  const unsigned grid = (unsigned)sparse_gather_blocks(t.N);
  const int R = t.R;
  if (R > kRankBlock) {
    if (loss_part)
      plca_rows_blocked_kernel<true><<<grid, 256, 0, st>>>(t.crow, t.col, t.val, Hz, W, R, t.N, P, norm, loss_part);
    else
      plca_rows_blocked_kernel<false><<<grid, 256, 0, st>>>(t.crow, t.col, t.val, Hz, W, R, t.N, P, norm, nullptr);
    NMF_LAUNCH_CHECK();
    return 0;
  }
  const int rpl = sparse_rpl(R);
#define PLCA_ROWS(RPLV)                                                                                                  \
  do {                                                                                                                   \
    if (loss_part)                                                                                                       \
      plca_rows_kernel<RPLV, true><<<grid, 256, 0, st>>>(t.crow, t.col, t.val, Hz, W, R, t.N, P, dHz, norm, loss_part); \
    else                                                                                                                 \
      plca_rows_kernel<RPLV, false><<<grid, 256, 0, st>>>(t.crow, t.col, t.val, Hz, W, R, t.N, P, dHz, norm, nullptr);  \
  } while (0)
  if (rpl <= 1) PLCA_ROWS(1);
  else if (rpl <= 2) PLCA_ROWS(2);
  else if (rpl <= 4) PLCA_ROWS(4);
  else PLCA_ROWS(8);
#undef PLCA_ROWS
  NMF_LAUNCH_CHECK();
  return 0;
}

int launch_gather(const int64_t* ptr, const int64_t* idx, const int64_t* perm, const float* P, const float* F, int R,
                  int64_t nseg, float* out, cudaStream_t st) {
  const dim3 grid((unsigned)sparse_gather_blocks(nseg), (unsigned)ceil_div(R, kRankBlock));
  const int rpl = R > kRankBlock ? 8 : sparse_rpl(R);
  if (rpl <= 1) plca_gather_kernel<1><<<grid, 256, 0, st>>>(ptr, idx, perm, P, F, R, nseg, out);
  else if (rpl <= 2) plca_gather_kernel<2><<<grid, 256, 0, st>>>(ptr, idx, perm, P, F, R, nseg, out);
  else if (rpl <= 4) plca_gather_kernel<4><<<grid, 256, 0, st>>>(ptr, idx, perm, P, F, R, nseg, out);
  else plca_gather_kernel<8><<<grid, 256, 0, st>>>(ptr, idx, perm, P, F, R, nseg, out);
  NMF_LAUNCH_CHECK();
  return 0;
}

int launch_colsum(const float* F, int64_t rows, int R, double* part, cudaStream_t st) {
  int64_t rpb;
  int nb;
  sparse_plca_colsum_plan(rows, &rpb, &nb);
  plca_colsum_part_kernel<<<dim3((unsigned)nb, (unsigned)ceil_div(R, 256)), 256, 0, st>>>(F, rows, R, rpb, part);
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace

void sparse_plca_colsum_plan(int64_t rows, int64_t* rpb, int* nb) {
  *rpb = ceil_div(rows, kColsumMaxBlocks);
  if (*rpb < 256) *rpb = 256;
  *nb = (int)ceil_div(rows, *rpb);
}

int64_t sparse_plca_loss_parts(int64_t N) { return sparse_gather_blocks(N); }

int64_t sparse_plca_colsum_parts(int64_t rows, int R) {
  int64_t rpb;
  int nb;
  sparse_plca_colsum_plan(rows, &rpb, &nb);
  return (int64_t)nb * R;
}

int sparse_plca_terms(const SparsePlcaTarget& t, const SparsePlcaWork& ws, const float* W, const float* Hz, float* dW,
                      float* dHz, float norm, double* loss_dev, cudaStream_t st) {
  const int R = t.R;
  // pass 1 (at R <= 256 with dHz), its loss partials when the loss is asked for
  int rc = launch_rows(t, W, Hz, ws.P, R > kRankBlock ? nullptr : dHz, norm, loss_dev ? ws.loss_part : nullptr, st);
  if (rc) return rc;
  if (dHz && R > kRankBlock && (rc = launch_gather(t.crow, t.col, nullptr, ws.P, W, R, t.N, dHz, st))) return rc;
  if (dW && (rc = launch_gather(t.ccol, t.row, t.perm, ws.P, Hz, R, t.C, dW, st))) return rc;
  if (!loss_dev) return 0;
  double* hpart = ws.cs_part + sparse_plca_colsum_parts(t.C, R);
  if ((rc = launch_colsum(W, t.C, R, ws.cs_part, st)) || (rc = launch_colsum(Hz, t.N, R, hpart, st))) return rc;
  int64_t rpb;
  int nbw, nbh;
  sparse_plca_colsum_plan(t.C, &rpb, &nbw);
  sparse_plca_colsum_plan(t.N, &rpb, &nbh);
  plca_loss_final_kernel<<<1, 256, 0, st>>>(ws.loss_part, sparse_plca_loss_parts(t.N), ws.cs_part, nbw, hpart, nbh, R,
                                            (double)norm, loss_dev);
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace nmfb200
