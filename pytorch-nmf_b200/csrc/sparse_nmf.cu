// Sparse-target NMF (reference: nmf.py:603-638 `_nmf_sp_recon_beta_pos_neg`, :95-119 `_sp_double_backward_update`): the
// numerators touch WH only at the non-zeros of V (SDDMM), and no kernel forms the dense N x C product.
//
//   beta 1:  num_H[n,:] = sum_{c in row n} v / (w_c . h_n + eps) * W[c,:]      den = colsum(W)                 nmf.py:617-619
//            num_W[c,:] = sum_{n in col c} v / (w_c . h_n + eps) * H[n,:]      den = colsum(H)
//            loss = V_norm + colsum(W) . colsum(H) - sum_nnz v log(w_c . h_n + eps)
//   beta 2:  num_H = V W, den_H = H (W^T W);  num_W = V^T H, den_W = W (H^T H)                                 nmf.py:608-611
//            loss = V_norm + 0.5 sum (H^T H o W^T W) - sum_nnz v (w_c . h_n)
//   other beta > 0 (x = w_c . h_n + eps):                                                                  nmf.py:621-636
//            num_H[n,:] = sum_{c in row n} v x^(beta-2) W[c,:]                den_H[n,:] = sum_c x^(beta-1) W[c,:] (all cells)
//            loss = V_norm + sum_all x^beta / beta - sum_nnz v x^(beta-1) / (beta-1),  V_norm = sum_nnz v^beta / (beta (beta-1))
//            The gathers here give the numerators and V_norm - neg; the V-free denominators and sum x^beta come from the fp32
//            contraction and loss kernels (simt_nmf.cu, kVFree), which never read V.
//
// One warp owns one segment -- a row of the CSR form (H update) or a column of the CSC form (W update) -- keeps its own factor
// row in registers, gathers the other factor's rows of its non-zeros (rank floats each, coalesced) and accumulates in fp32 in
// the order of the stored indices: deterministic, no atomics.
//
// Observed cells (nmfb200_nmf_set_target_observed): the stored entries are the observed cells of a masked fit, zeros
// included, and the loss is beta_div(WH[obs], V[obs]) at every beta.  Both backward passes of that loss are sums over the
// observed cells only, so ONE gather per segment forms both terms, with x = w_j . f_s and a(x), b(x) of nmf.py:61-74:
//   num[s,:] = sum_j v a(x) w_j      den[s,:] = sum_j b(x) w_j
//   beta 2: a = 1, b = x;  beta 1: a = 1 / (x + eps), b = 1;  beta 0: a = 1 / (x + eps)^2, b = 1 / (x + eps);
//   other:  b = (x + eps)^(beta - 1) from one powf, a = b / (x + eps)
// and the loss gather sums metrics.beta_div's per-cell term (loss_term) at each stored entry, in double.  A weighted fit
// (nmfb200_nmf_set_target_observed_weighted) reads one weight w per entry beside its value, in the same order:
//   num[s,:] = sum_j (w v) a(x) w_j      den[s,:] = sum_j (w b(x)) w_j      loss = sum_j w loss_term
#include "common.cuh"

namespace nmfb200 {

namespace {

enum SpMode : int { kSpKL = 0, kSpEU = 1, kSpKLLoss = 2, kSpEULoss = 3, kSpBeta = 4, kSpBetaLoss = 5, kSpObsTerms = 6,
                    kSpObsLoss = 7 };
constexpr int kSpGramPass = 256 * 16;                 // Gram pairs per pass of sp_gram_part_kernel (16 per thread)

// a(x) and b(x) of an observed cell at beta mode BM (BetaMode), x = w_j . f_s; bm1 = beta - 1 (kGeneric only)
template <int BM>
__device__ __forceinline__ void obs_phi(float x, float bm1, float& a, float& b) {
  if (BM == kEU) {
    a = 1.f;
    b = x;                                                // nmf.py:62-63 (no eps)
  } else if (BM == kKL) {
    a = 1.0f / (x + kEps);                                // nmf.py:65; den: the observed cells' rows of the other factor
    b = 1.f;
  } else if (BM == kIS) {
    const float r = 1.0f / (x + kEps);                    // nmf.py:68-70
    a = r * r;
    b = r;
  } else {
    const float xe = x + kEps;                            // nmf.py:72-74
    b = powf(xe, bm1);
    a = b / xe;
  }
}

// pa, pb, ca, cb: the beta constants of kSpBeta / kSpBetaLoss (unused by the other modes); kSpObsTerms: pa = beta - 1,
// den_out the denominator (nseg x R); kSpObsLoss: pa = beta.  BM: the beta mode of the two observed-cell modes; WT: they
// read the entries' weights wt (in val's order).
template <int RPL, int MODE, int BM = kKL, bool WT = false>
__device__ __forceinline__ void
sp_gather(const int64_t* __restrict__ ptr, const int64_t* __restrict__ idx, const float* __restrict__ val,
          const float* __restrict__ Fs, const float* __restrict__ Fo, int R, int64_t nseg, float* __restrict__ out,
          float* __restrict__ den_out, double* __restrict__ loss_part, float pa, float pb, double ca, double cb,
          const float* __restrict__ wt = nullptr) {
  const int lane = threadIdx.x & 31;
  const int64_t seg = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  double lacc = 0.0;
  if (seg < nseg) {
    float hs[RPL], acc[RPL], dacc[RPL];
#pragma unroll
    for (int k = 0; k < RPL; ++k) {
      const int r = lane + 32 * k;
      hs[k] = r < R ? Fs[seg * R + r] : 0.f;
      acc[k] = 0.f;
      dacc[k] = 0.f;
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
      } else if (MODE == kSpBeta) {
        const float ratio = v * powf(dot + kEps, pa);                 // pa = beta - 2: phi<kGeneric>'s pn at a stored entry
#pragma unroll
        for (int k = 0; k < RPL; ++k) acc[k] = fmaf(ratio, w[k], acc[k]);
      } else if (MODE == kSpBetaLoss) {
        // pa = beta, pb = beta - 1, ca = 1 / (beta (beta - 1)), cb = 1 / (beta - 1): V_norm's and neg's terms of this entry
        lacc += (double)powf(v, pa) * ca - (double)(v * powf(dot + kEps, pb)) * cb;
      } else if (MODE == kSpObsTerms) {
        float a, b;
        obs_phi<BM>(dot, pa, a, b);
        float ratio;
        if constexpr (WT) {
          const float we = wt[e];
          ratio = (we * v) * a;
          b = we * b;
        } else {
          ratio = v * a;
        }
#pragma unroll
        for (int k = 0; k < RPL; ++k) {
          acc[k] = fmaf(ratio, w[k], acc[k]);
          dacc[k] = fmaf(b, w[k], dacc[k]);
        }
      } else if (MODE == kSpObsLoss) {
        if constexpr (WT) lacc += (double)(wt[e] * loss_term<BM>(v, dot, pa));
        else lacc += (double)loss_term<BM>(v, dot, pa);              // metrics.py:60-96 at this cell
      } else if (MODE == kSpKLLoss) {
        lacc += (double)(v * logf(dot + kEps));                      // nmf.py:619
      } else {
        lacc += (double)(v * dot);                                   // nmf.py:610
      }
    }
    if (MODE == kSpKL || MODE == kSpEU || MODE == kSpBeta || MODE == kSpObsTerms) {
#pragma unroll
      for (int k = 0; k < RPL; ++k) {
        const int r = lane + 32 * k;
        if (r < R) out[seg * R + r] = acc[k];
        if (MODE == kSpObsTerms && r < R) den_out[seg * R + r] = dacc[k];
      }
    }
  }
  if (MODE == kSpKLLoss || MODE == kSpEULoss || MODE == kSpBetaLoss || MODE == kSpObsLoss) {
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

template <int RPL, int MODE>
__global__ void __launch_bounds__(256)
sp_gather_kernel(const int64_t* __restrict__ ptr, const int64_t* __restrict__ idx, const float* __restrict__ val,
                 const float* __restrict__ Fs, const float* __restrict__ Fo, int R, int64_t nseg, float* __restrict__ out,
                 double* __restrict__ loss_part) {
  sp_gather<RPL, MODE>(ptr, idx, val, Fs, Fo, R, nseg, out, nullptr, loss_part, 0.f, 0.f, 0.0, 0.0);
}

// the modes of beta != 1, 2, with their constants
template <int RPL, int MODE>
__global__ void __launch_bounds__(256)
sp_gather_beta_kernel(const int64_t* __restrict__ ptr, const int64_t* __restrict__ idx, const float* __restrict__ val,
                      const float* __restrict__ Fs, const float* __restrict__ Fo, int R, int64_t nseg, float* __restrict__ out,
                      double* __restrict__ loss_part, float pa, float pb, double ca, double cb) {
  sp_gather<RPL, MODE>(ptr, idx, val, Fs, Fo, R, nseg, out, nullptr, loss_part, pa, pb, ca, cb);
}

// the observed-cell modes (kSpObsTerms, kSpObsLoss) at beta mode BM; pa as sp_gather's; WT: with the entries' weights wt
template <int RPL, int MODE, int BM, bool WT>
__global__ void __launch_bounds__(256)
sp_gather_obs_kernel(const int64_t* __restrict__ ptr, const int64_t* __restrict__ idx, const float* __restrict__ val,
                     const float* __restrict__ Fs, const float* __restrict__ Fo, int R, int64_t nseg, float* __restrict__ num,
                     float* __restrict__ den, double* __restrict__ loss_part, float pa, const float* __restrict__ wt) {
  sp_gather<RPL, MODE, BM, WT>(ptr, idx, val, Fs, Fo, R, nseg, num, den, loss_part, pa, 0.f, 0.0, 0.0, wt);
}

// Gram matrix G = F^T F (R x R) of a (rows x R) factor: per-block slabs, then a fixed-order sum over the blocks.
// BATCH: bt.n problems, problem b's F at F + b bt.f, on the single problem's nb blocks [b nb, (b + 1) nb) of grid x; the
// slabs stay indexed by blockIdx.x, so problem b's are the b-th run of nb.  The single-problem instantiations compile none of it.
template <bool BATCH>
__global__ void __launch_bounds__(256)
sp_gram_part_kernel(const float* __restrict__ F, int64_t rows, int R, int64_t rpb, float* __restrict__ part, Batch bt) {
  extern __shared__ float tile[];                     // [32][R]
  int64_t bx = blockIdx.x;
  if constexpr (BATCH) {
    const int64_t nb = gridDim.x / bt.n;
    const int64_t prob = bx / nb;
    if (batch_skips(bt.active, prob)) return;
    bx -= prob * nb;
    F += prob * bt.f;
  }
  const int64_t r0 = bx * rpb, r1 = min(rows, r0 + rpb);
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

// BATCH: problem b sums its own run of nb slabs into out + b bt.p, on the single problem's ceil(n / 256) blocks of grid x
template <bool BATCH>
__global__ void sp_gram_sum_kernel(const float* __restrict__ part, int nb, int n, float* __restrict__ out, Batch bt) {
  int p;
  if constexpr (BATCH) {
    const int64_t nbx = (n + 255) / 256;
    const int64_t prob = (int64_t)blockIdx.x / nbx;
    if (batch_skips(bt.active, prob)) return;
    p = (int)((int64_t)blockIdx.x - prob * nbx) * 256 + threadIdx.x;
    part += prob * nb * (int64_t)n;
    out += prob * bt.p;
  } else {
    p = blockIdx.x * 256 + threadIdx.x;
  }
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

// loss = (v_norm - neg) + pos / beta at beta != 1, 2: the gather's partials and the V-free sum x^beta's, each summed in a fixed
// order (one block, strided per thread, then a fixed tree)
__global__ void __launch_bounds__(256)
sp_beta_loss_final_kernel(const double* __restrict__ vn_neg_part, int nvn, const double* __restrict__ pos_part, int npos,
                          double beta, double* __restrict__ out) {
  __shared__ double sa[256], sb[256];
  double a = 0.0, b = 0.0;
  for (int i = threadIdx.x; i < nvn; i += 256) a += vn_neg_part[i];
  for (int i = threadIdx.x; i < npos; i += 256) b += pos_part[i];
  sa[threadIdx.x] = a;
  sb[threadIdx.x] = b;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) { sa[threadIdx.x] += sa[threadIdx.x + o]; sb[threadIdx.x] += sb[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sa[0] + sb[0] / beta;                 // nmf.py:635: pos /= beta
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
                  int64_t nseg, float* out, double* loss_part, cudaStream_t st, float pa = 0.f, float pb = 0.f,
                  double ca = 0.0, double cb = 0.0) {
  const unsigned grid = (unsigned)sparse_gather_blocks(nseg);
  const int rpl = sparse_rpl(R);
#define NMF_GATHER(RPLV)                                                                                           \
  do {                                                                                                             \
    if constexpr (MODE == kSpBeta || MODE == kSpBetaLoss)                                                          \
      sp_gather_beta_kernel<RPLV, MODE><<<grid, 256, 0, st>>>(ptr, idx, val, Fs, Fo, R, nseg, out, loss_part, pa, pb, \
                                                              ca, cb);                                             \
    else                                                                                                           \
      sp_gather_kernel<RPLV, MODE><<<grid, 256, 0, st>>>(ptr, idx, val, Fs, Fo, R, nseg, out, loss_part);           \
  } while (0)
  if (rpl <= 1) NMF_GATHER(1);
  else if (rpl <= 2) NMF_GATHER(2);
  else if (rpl <= 4) NMF_GATHER(4);
  else NMF_GATHER(8);
#undef NMF_GATHER
  NMF_LAUNCH_CHECK();
  return 0;
}

// The observed-cell gathers: MODE kSpObsTerms or kSpObsLoss, on the plan of launch_gather; wt (optional) the entries' weights
template <int MODE>
int launch_observed(const int64_t* ptr, const int64_t* idx, const float* val, const float* Fs, const float* Fo, int R,
                    int64_t nseg, double beta, float* num, float* den, double* loss_part, cudaStream_t st,
                    const float* wt) {
  const unsigned grid = (unsigned)sparse_gather_blocks(nseg);
  const int rpl = sparse_rpl(R);
  const float pa = (float)(MODE == kSpObsTerms ? beta - 1.0 : beta);
  auto go = [&](auto bm, auto weighted) {
    constexpr int BM = decltype(bm)::value;
    constexpr bool WT = decltype(weighted)::value;
#define NMF_OBS(RPLV) \
  sp_gather_obs_kernel<RPLV, MODE, BM, WT><<<grid, 256, 0, st>>>(ptr, idx, val, Fs, Fo, R, nseg, num, den, loss_part, pa, wt)
    if (rpl <= 1) NMF_OBS(1);
    else if (rpl <= 2) NMF_OBS(2);
    else if (rpl <= 4) NMF_OBS(4);
    else NMF_OBS(8);
#undef NMF_OBS
  };
  auto by_beta = [&](auto weighted) {
    switch (beta_mode(beta)) {
      case kKL: go(std::integral_constant<int, kKL>{}, weighted); break;
      case kEU: go(std::integral_constant<int, kEU>{}, weighted); break;
      case kIS: go(std::integral_constant<int, kIS>{}, weighted); break;
      default: go(std::integral_constant<int, kGeneric>{}, weighted); break;
    }
  };
  if (wt) by_beta(std::true_type{});
  else by_beta(std::false_type{});
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace

int64_t sparse_gram_part_floats(int R) { return (int64_t)128 * R * R; }

// raw numerator of one factor update: out (nseg x R); ptr / idx / val = the compressed form whose segments are that factor's rows
int sparse_numerator(const int64_t* ptr, const int64_t* idx, const float* val, const float* Fself, const float* Fother,
                     int R, int64_t nseg, double beta, float* out, cudaStream_t st) {
  if (beta == 1.0) return launch_gather<kSpKL>(ptr, idx, val, Fself, Fother, R, nseg, out, nullptr, st);
  if (beta == 2.0) return launch_gather<kSpEU>(ptr, idx, val, Fself, Fother, R, nseg, out, nullptr, st);
  return launch_gather<kSpBeta>(ptr, idx, val, Fself, Fother, R, nseg, out, nullptr, st, (float)(beta - 2.0));
}

int sparse_gram(const float* F, int64_t rows, int R, float* part, float* out, cudaStream_t st, const Batch& bt) {
  int64_t rpb;
  int nb;
  sparse_gram_plan(rows, &rpb, &nb);
  const int64_t nsum = ceil_div((int64_t)R * R, 256);
  if (bt.n < 1 || nb > kMaxGridX / bt.n || nsum > kMaxGridX / bt.n) {
    set_error("sparse_gram: batch x blocks pass grid x");
    return 1;
  }
  const size_t smem = 32 * R * sizeof(float);
  if (bt.n > 1 || bt.active) {
    sp_gram_part_kernel<true><<<(unsigned)(nb * bt.n), 256, smem, st>>>(F, rows, R, rpb, part, bt);
    NMF_LAUNCH_CHECK();
    sp_gram_sum_kernel<true><<<(unsigned)(nsum * bt.n), 256, 0, st>>>(part, nb, R * R, out, bt);
  } else {
    sp_gram_part_kernel<false><<<nb, 256, smem, st>>>(F, rows, R, rpb, part, bt);
    NMF_LAUNCH_CHECK();
    sp_gram_sum_kernel<false><<<(unsigned)nsum, 256, 0, st>>>(part, nb, R * R, out, bt);
  }
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

int sparse_beta_loss(const int64_t* crow, const int64_t* col, const float* val, const float* H, const float* W, int R,
                     int64_t N, double beta, const double* pos_part, int npos, double* loss_part, double* loss_dev,
                     cudaStream_t st) {
  int rc = launch_gather<kSpBetaLoss>(crow, col, val, H, W, R, N, nullptr, loss_part, st, (float)beta, (float)(beta - 1.0),
                                      1.0 / (beta * (beta - 1.0)), 1.0 / (beta - 1.0));
  if (rc) return rc;
  sp_beta_loss_final_kernel<<<1, 256, 0, st>>>(loss_part, (int)sparse_gather_blocks(N), pos_part, npos, beta, loss_dev);
  NMF_LAUNCH_CHECK();
  return 0;
}

// Observed cells: both raw terms of one factor's update (num, den: nseg x R) over the compressed form whose segments are that
// factor's rows
int observed_terms(const int64_t* ptr, const int64_t* idx, const float* val, const float* Fself, const float* Fother, int R,
                   int64_t nseg, double beta, float* num, float* den, cudaStream_t st, const float* wt) {
  return launch_observed<kSpObsTerms>(ptr, idx, val, Fself, Fother, R, nseg, beta, num, den, nullptr, st, wt);
}

// Observed cells: loss_dev = sum over the stored entries of metrics.beta_div's term, one partial per block over the CSR rows,
// then a fixed-order sum
int observed_loss(const int64_t* crow, const int64_t* col, const float* val, const float* H, const float* W, int R, int64_t N,
                  double beta, double* loss_part, double* loss_dev, cudaStream_t st, const float* wt) {
  int rc = launch_observed<kSpObsLoss>(crow, col, val, H, W, R, N, beta, nullptr, nullptr, loss_part, st, wt);
  if (rc) return rc;
  // no V-free part: npos = 0, and the divisor 1 leaves the gather's sum as it is (at every beta, 0 included)
  sp_beta_loss_final_kernel<<<1, 256, 0, st>>>(loss_part, (int)sparse_gather_blocks(N), nullptr, 0, 1.0, loss_dev);
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace nmfb200
