// Sparse-target NMF (reference: nmf.py:603-638 `_nmf_sp_recon_beta_pos_neg`, :95-119 `_sp_double_backward_update`), beta 1 and 2:
// the update terms touch WH only at the non-zeros of V (SDDMM) and never form the dense N x C product.
//
//   beta 1:  num_H[n,:] = sum_{c in row n} v / (w_c . h_n + eps) * W[c,:]      den = colsum(W)                 nmf.py:617-619
//            num_W[c,:] = sum_{n in col c} v / (w_c . h_n + eps) * H[n,:]      den = colsum(H)
//            loss = V_norm + colsum(W) . colsum(H) - sum_nnz v log(w_c . h_n + eps)
//   beta 2:  num_H = V W, den_H = H (W^T W);  num_W = V^T H, den_W = W (H^T H)                                 nmf.py:608-611
//            loss = V_norm + 0.5 sum (H^T H o W^T W) - sum_nnz v (w_c . h_n)
//
// One warp owns one segment -- a row of the CSR form (H update) or a column of the CSC form (W update) -- keeps its own factor
// row in registers, gathers the other factor's rows of its non-zeros (rank floats each, coalesced) and accumulates in fp32 in
// the order of the stored indices: deterministic, no atomics.
#include "common.cuh"

namespace nmfb200 {

namespace {

enum SpMode : int { kSpKL = 0, kSpEU = 1, kSpKLLoss = 2, kSpEULoss = 3 };
constexpr int kSpGramPass = 256 * 16;                 // Gram pairs per pass of sp_gram_part_kernel (16 per thread)

template <int RPL, int MODE>
__global__ void __launch_bounds__(256)
sp_gather_kernel(const int64_t* __restrict__ ptr, const int64_t* __restrict__ idx, const float* __restrict__ val,
                 const float* __restrict__ Fs, const float* __restrict__ Fo, int R, int64_t nseg, float* __restrict__ out,
                 double* __restrict__ loss_part) {
  const int lane = threadIdx.x & 31;
  const int64_t seg = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  double lacc = 0.0;
  if (seg < nseg) {
    float hs[RPL], acc[RPL];
#pragma unroll
    for (int k = 0; k < RPL; ++k) {
      const int r = lane + 32 * k;
      hs[k] = r < R ? Fs[seg * R + r] : 0.f;
      acc[k] = 0.f;
    }
    const int64_t e0 = ptr[seg], e1 = ptr[seg + 1];
    for (int64_t e = e0; e < e1; ++e) {
      const int64_t j = idx[e];
      const float v = val[e];
      float w[RPL];
#pragma unroll
      for (int k = 0; k < RPL; ++k) {
        const int r = lane + 32 * k;
        w[k] = r < R ? Fo[j * R + r] : 0.f;
      }
      float dot = 0.f;
      if (MODE != kSpEU) {
#pragma unroll
        for (int k = 0; k < RPL; ++k) dot = fmaf(w[k], hs[k], dot);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
      }
      if (MODE == kSpKL) {
        const float ratio = v / (dot + kEps);                        // nmf.py:619 (derivative of v log(WH + eps))
#pragma unroll
        for (int k = 0; k < RPL; ++k) acc[k] = fmaf(ratio, w[k], acc[k]);
      } else if (MODE == kSpEU) {
#pragma unroll
        for (int k = 0; k < RPL; ++k) acc[k] = fmaf(v, w[k], acc[k]);
      } else if (MODE == kSpKLLoss) {
        lacc += (double)(v * logf(dot + kEps));                      // nmf.py:619
      } else {
        lacc += (double)(v * dot);                                   // nmf.py:610
      }
    }
    if (MODE == kSpKL || MODE == kSpEU) {
#pragma unroll
      for (int k = 0; k < RPL; ++k) {
        const int r = lane + 32 * k;
        if (r < R) out[seg * R + r] = acc[k];
      }
    }
  }
  if (MODE == kSpKLLoss || MODE == kSpEULoss) {
    __shared__ double sh[8];
    if (lane == 0) sh[threadIdx.x >> 5] = lacc;       // every lane holds the same sum
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int k = 0; k < 8; ++k) t += sh[k];
      loss_part[blockIdx.x] = t;
    }
  }
}

// Gram matrix G = F^T F (R x R) of a (rows x R) factor: per-block slabs, then a fixed-order sum over the blocks
__global__ void __launch_bounds__(256)
sp_gram_part_kernel(const float* __restrict__ F, int64_t rows, int R, int64_t rpb, float* __restrict__ part) {
  extern __shared__ float tile[];                     // [32][R]
  const int64_t r0 = (int64_t)blockIdx.x * rpb, r1 = min(rows, r0 + rpb);
  const int npairs = R * R;
  float acc[16];                                      // R <= 64: 4096 / 256; larger ranks loop below
  for (int base = 0; base < npairs; base += kSpGramPass) {
#pragma unroll
    for (int k = 0; k < 16; ++k) acc[k] = 0.f;
    for (int64_t rr = r0; rr < r1; rr += 32) {
      const int nrow = (int)min((int64_t)32, r1 - rr);
      __syncthreads();
      for (int i = threadIdx.x; i < nrow * R; i += 256) tile[i] = F[rr * R + i];
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const int p = base + threadIdx.x + 256 * k;
        if (p < npairs) {
          const int a = p / R, b = p - a * R;
          float s = 0.f;
          for (int q = 0; q < nrow; ++q) s = fmaf(tile[q * R + a], tile[q * R + b], s);
          acc[k] += s;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int p = base + threadIdx.x + 256 * k;
      if (p < npairs) part[(int64_t)blockIdx.x * npairs + p] = acc[k];
    }
  }
}

__global__ void sp_gram_sum_kernel(const float* __restrict__ part, int nb, int n, float* __restrict__ out) {
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= n) return;
  float s = 0.f;
  for (int b = 0; b < nb; ++b) s += part[(int64_t)b * n + p];
  out[p] = s;
}

// den[row,:] = F[row,:] G  (G: R x R), one warp per row
template <int RPL>
__global__ void __launch_bounds__(256)
sp_rows_times_gram_kernel(const float* __restrict__ F, const float* __restrict__ G, int64_t rows, int R, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  float f[RPL], acc[RPL];
#pragma unroll
  for (int k = 0; k < RPL; ++k) { const int r = lane + 32 * k; f[k] = r < R ? F[row * R + r] : 0.f; acc[k] = 0.f; }
  for (int i = 0; i < R; ++i) {
    const float fi = __shfl_sync(0xffffffffu, f[i >> 5], i & 31);
#pragma unroll
    for (int k = 0; k < RPL; ++k) { const int r = lane + 32 * k; if (r < R) acc[k] = fmaf(fi, G[i * R + r], acc[k]); }
  }
#pragma unroll
  for (int k = 0; k < RPL; ++k) { const int r = lane + 32 * k; if (r < R) out[row * R + r] = acc[k]; }
}

// loss = v_norm + pos - neg:  beta 1: pos = colsum(W) . colsum(H);  beta 2: pos = 0.5 sum(GW o GH)
__global__ void sp_loss_final_kernel(const double* __restrict__ neg_part, int nparts, const float* __restrict__ a,
                                     const float* __restrict__ b, int n, double scale, double v_norm, double* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double neg = 0.0, pos = 0.0;
  for (int i = 0; i < nparts; ++i) neg += neg_part[i];
  for (int i = 0; i < n; ++i) pos += (double)a[i] * (double)b[i];
  *out = v_norm + scale * pos - neg;
}

}  // namespace

// Launch plans, shared by the launchers below and by nmfb200_nmf_sparse_plan.
// Rank floats per lane of the warp-per-segment kernels: 1, 2, 4 or 8 (R <= 32, 64, 128, 256).
int sparse_rpl(int R) {
  const int rpl = (R + 31) / 32;
  return rpl <= 1 ? 1 : rpl <= 2 ? 2 : rpl <= 4 ? 4 : 8;
}
// Blocks of the warp-per-segment kernels (8 warps each) over nseg segments or rows.
int64_t sparse_gather_blocks(int64_t nseg) { return ceil_div(nseg, 8); }
// Gram of a rows x R factor: at most 128 blocks of rpb rows (a multiple of the 32-row slab), the last one possibly short.
void sparse_gram_plan(int64_t rows, int64_t* rpb, int* nb) {
  *rpb = round_up(ceil_div(rows, 128), 32);
  *nb = (int)ceil_div(rows, *rpb);
}
int sparse_gram_passes(int R) { return (int)ceil_div((int64_t)R * R, kSpGramPass); }

namespace {

template <int MODE>
int launch_gather(const int64_t* ptr, const int64_t* idx, const float* val, const float* Fs, const float* Fo, int R,
                  int64_t nseg, float* out, double* loss_part, cudaStream_t st) {
  const unsigned grid = (unsigned)sparse_gather_blocks(nseg);
  const int rpl = sparse_rpl(R);
  if (rpl <= 1) sp_gather_kernel<1, MODE><<<grid, 256, 0, st>>>(ptr, idx, val, Fs, Fo, R, nseg, out, loss_part);
  else if (rpl <= 2) sp_gather_kernel<2, MODE><<<grid, 256, 0, st>>>(ptr, idx, val, Fs, Fo, R, nseg, out, loss_part);
  else if (rpl <= 4) sp_gather_kernel<4, MODE><<<grid, 256, 0, st>>>(ptr, idx, val, Fs, Fo, R, nseg, out, loss_part);
  else sp_gather_kernel<8, MODE><<<grid, 256, 0, st>>>(ptr, idx, val, Fs, Fo, R, nseg, out, loss_part);
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace

int64_t sparse_gram_part_floats(int R) { return (int64_t)128 * R * R; }

// raw numerator of one factor update: out (nseg x R); ptr / idx / val = the compressed form whose segments are that factor's rows
int sparse_numerator(const int64_t* ptr, const int64_t* idx, const float* val, const float* Fself, const float* Fother,
                     int R, int64_t nseg, double beta, float* out, cudaStream_t st) {
  if (beta == 1.0) return launch_gather<kSpKL>(ptr, idx, val, Fself, Fother, R, nseg, out, nullptr, st);
  return launch_gather<kSpEU>(ptr, idx, val, Fself, Fother, R, nseg, out, nullptr, st);
}

int sparse_gram(const float* F, int64_t rows, int R, float* part, float* out, cudaStream_t st) {
  int64_t rpb;
  int nb;
  sparse_gram_plan(rows, &rpb, &nb);
  sp_gram_part_kernel<<<nb, 256, 32 * R * sizeof(float), st>>>(F, rows, R, rpb, part);
  NMF_LAUNCH_CHECK();
  sp_gram_sum_kernel<<<(unsigned)ceil_div(R * R, 256), 256, 0, st>>>(part, nb, R * R, out);
  NMF_LAUNCH_CHECK();
  return 0;
}

int sparse_rows_times_gram(const float* F, const float* G, int64_t rows, int R, float* out, cudaStream_t st) {
  const unsigned grid = (unsigned)sparse_gather_blocks(rows);
  const int rpl = sparse_rpl(R);
  if (rpl <= 1) sp_rows_times_gram_kernel<1><<<grid, 256, 0, st>>>(F, G, rows, R, out);
  else if (rpl <= 2) sp_rows_times_gram_kernel<2><<<grid, 256, 0, st>>>(F, G, rows, R, out);
  else if (rpl <= 4) sp_rows_times_gram_kernel<4><<<grid, 256, 0, st>>>(F, G, rows, R, out);
  else sp_rows_times_gram_kernel<8><<<grid, 256, 0, st>>>(F, G, rows, R, out);
  NMF_LAUNCH_CHECK();
  return 0;
}

// loss_dev = v_norm + pos - neg over the CSR form (rows of H); pos_a / pos_b: the two colsum vectors (beta 1, n = R, scale 1)
// or the two Gram matrices (beta 2, n = R * R, scale 0.5)
int sparse_loss(const int64_t* crow, const int64_t* col, const float* val, const float* H, const float* W, int R, int64_t N,
                double beta, const float* pos_a, const float* pos_b, double v_norm, double* loss_part, double* loss_dev,
                cudaStream_t st) {
  int rc = beta == 1.0 ? launch_gather<kSpKLLoss>(crow, col, val, H, W, R, N, nullptr, loss_part, st)
                       : launch_gather<kSpEULoss>(crow, col, val, H, W, R, N, nullptr, loss_part, st);
  if (rc) return rc;
  sp_loss_final_kernel<<<1, 32, 0, st>>>(loss_part, (int)sparse_gather_blocks(N), pos_a, pos_b, beta == 1.0 ? R : R * R,
                                         beta == 1.0 ? 1.0 : 0.5, v_norm, loss_dev);
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace nmfb200
