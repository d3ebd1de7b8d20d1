// Coordinate descent at beta 2 on the observed cells of a target (nmfb200_nmf_observed_cd_update): CCD++ of Yu et al.
// 2012, made non-negative, on the compressed forms nmfb200_nmf_set_target_observed registers.
//
// One factor update of  1/2 sum_{(n,c) in O} w (v - h_n . w_c)^2 + l1 (sum W + sum H) + l2 / 2 (|W|^2 + |H|^2)  with the
// other factor F fixed.  Every row s of the updated factor X runs on its own, over the observed cells O_s of its segment (a
// column of V, CSC, for W; a row of V, CSR, for H): with r = v - F x_s on O_s at the current x_s,
//   for k = 0 .. R-1:  num = sum_{j in O_s} w_j r_j f_{j,k},  hess = sum_{j in O_s} w_j f_{j,k}^2 + l2,
//                      if hess != 0:  x_{s,k} <- max(0, x_{s,k} + (num - l1 - l2 x_{s,k}) / hess)
// (w = 1 without weights).  With every cell observed and unit weights this is cd.cu's HALS update in exact arithmetic.
//
// One warp owns one segment and keeps its x_s in registers (lane l: components l, l + 32, ...).  The components go in
// groups of 32, one per lane.  For group g, ONE pass over the segment's entries, in stored order, reads each entry's
// 32-float slice f_j[32g .. 32g + 31] (coalesced) and forms
//   a_l = sum_j w r_j f_{j,32g+l}   and   G[i,l] = sum_j w f_{j,32g+i} f_{j,32g+l}   (lane l: column l, from shuffles),
// with r at the start of the group.  The group is then swept in registers as cd.cu sweeps a row:
//   num_k = a_k - sum_{i<k} delta_i G[i,k],  hess = G[k,k] + l2,  delta_k = x_new - x_old,
// since the residual after the group's earlier steps is r - sum_{i<k} delta_i f_{j,i}.  The residual enters group 0 as
// v - x_s . f_j (a full-rank dot in the pass), and group g > 0 takes it from the previous group's pass, less
// sum_i delta_i f_{j,32(g-1)+i} of the previous group's steps (computed in group g's pass).  For R <= 32 there is one group
// and r is never stored; above, it lives in an O(observed) fp32 workspace indexed by the entry (`rbuf`).
//
// Summation orders (fixed by the segment's stored order and R alone, whatever the grid; the oracle tolerance rests on them):
//   x_s . f_j and sum_i delta_i f_{j,i}: lane l accumulates its components l, l + 32, ... in ascending order with fmaf from
//           0, then the 32 lane sums are added by an xor butterfly over lane distances 16, 8, 4, 2, 1;
//   a_l, G[i,l]: one fmaf per entry in stored order from 0, the weight applied first (w r, w f_{j,32g+l});
//   sum_{i<k} delta_i G[i,k]: lane k accumulates i = 0, 1, ..., k - 1 with fmaf from 0.
// No atomics: a run is bit for bit repeatable.
//
// Cost per factor update: one pass per group, ceil(R / 32) passes over the observed entries, each reading 32 floats of
// f_j per entry (the first pass all R of them, the later ones the previous group's slice too).  A segment is one warp's
// work however long it is: on a skewed distribution the few longest segments set the tail of the launch, as they do for
// the observed-cell gathers of sparse_nmf.cu.
#include "common.cuh"

namespace nmfb200 {

namespace {

constexpr int kSegsPerBlock = 8;   // one warp per segment

__device__ __forceinline__ float warp_sum(float p) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
  return p;
}

// RPL: rank floats per lane (R <= 32 RPL); WT: the entries carry weights wt (in val's order).  ptr / idx / val: the
// compressed form whose segments are X's rows; X (nseg x R) is updated in place, F (rows of idx x R) is read.  FIXED: the
// components k with fixed[k] != 0 take no step (delta 0), so the residual the later components see is unchanged.
template <int RPL, bool WT, bool FIXED = false>
__global__ void __launch_bounds__(256)
observed_cd_kernel(const int64_t* __restrict__ ptr, const int64_t* __restrict__ idx, const float* __restrict__ val,
                   const float* __restrict__ wt, float* __restrict__ X, const float* __restrict__ F, int R, int64_t nseg,
                   float* __restrict__ rbuf, float l1, float l2, const uint8_t* __restrict__ fixed) {
  const int lane = threadIdx.x & 31;
  const int64_t seg = (int64_t)blockIdx.x * kSegsPerBlock + (threadIdx.x >> 5);
  if (seg >= nseg) return;                       // the whole warp leaves together
  float x[RPL];
#pragma unroll
  for (int m = 0; m < RPL; ++m) {
    const int k = lane + 32 * m;
    x[m] = k < R ? X[seg * R + k] : 0.f;
  }
  const int64_t e0 = ptr[seg], e1 = ptr[seg + 1];
  const int ngroups = (R + 31) / 32;
  float dprev = 0.f;                             // this lane's delta in the previous group

#pragma unroll
  for (int g = 0; g < RPL; ++g) {
    if (g < ngroups) {
      const int kg = lane + 32 * g;
      float a = 0.f, G[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) G[i] = 0.f;
      for (int64_t e = e0; e < e1; ++e) {
        const float* fj = F + idx[e] * R;
        float r, f;
        if (g == 0) {
          float fr[RPL];
          float p = 0.f;
#pragma unroll
          for (int m = 0; m < RPL; ++m) {
            const int k = lane + 32 * m;
            fr[m] = k < R ? fj[k] : 0.f;
            p = fmaf(x[m], fr[m], p);
          }
          r = val[e] - warp_sum(p);
          f = fr[0];
        } else {
          const int kp = kg - 32;
          const float fp = fj[kp];               // kp < R: the previous group is full
          // lane 0 alone reads and writes rbuf[e]: no lane reads it after the write
          const float rin = __shfl_sync(0xffffffffu, lane == 0 ? rbuf[e] : 0.f, 0);
          r = rin - warp_sum(dprev * fp);
          f = kg < R ? fj[kg] : 0.f;
        }
        if (g + 1 < ngroups && lane == 0) rbuf[e] = r;
        float wr = r, wf = f;
        if constexpr (WT) {
          const float w = wt[e];
          wr = w * r;
          wf = w * f;
        }
        a = fmaf(wr, f, a);
#pragma unroll
        for (int i = 0; i < 32; ++i) G[i] = fmaf(wf, __shfl_sync(0xffffffffu, f, i), G[i]);
      }
      // the sweep of the group: lane k owns component 32 g + k; corr = sum_{i<k} delta_i G[i, lane]
      const int kend = min(32, R - 32 * g);
      float corr = 0.f, mine = 0.f;
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        if (k < kend) {
          float d = 0.f;
          if (lane == k) {
            const float hess = G[k] + l2;
            if (hess != 0.f && !(FIXED && fixed[32 * g + k])) {   // a dead or fixed component keeps its value, as in cd.cu
              const float xo = x[g];
              const float xn = fmaxf(0.f, xo + (a - corr - l1 - l2 * xo) / hess);
              x[g] = xn;
              d = xn - xo;
            }
            mine = d;
          }
          d = __shfl_sync(0xffffffffu, d, k);
          corr = fmaf(d, G[k], corr);
        }
      }
      dprev = mine;
    }
  }

#pragma unroll
  for (int m = 0; m < RPL; ++m) {
    const int k = lane + 32 * m;
    if (k < R) X[seg * R + k] = x[m];
  }
}

}  // namespace

int64_t observed_cd_workspace_floats(int R, int64_t nnz) { return R > 32 ? nnz : 0; }

int observed_cd(const int64_t* ptr, const int64_t* idx, const float* val, const float* wt, float* X, const float* F, int R,
                int64_t nseg, float* rbuf, float l1, float l2, cudaStream_t st, const uint8_t* fixed) {
  if (R < 1 || R > 256) { set_error("observed_cd: rank must be in [1, 256]"); return 1; }
  if (nseg < 1) return 0;
  const int64_t blocks = ceil_div(nseg, (int64_t)kSegsPerBlock);
  if (blocks > kMaxGridX) { set_error("observed_cd: segment blocks pass grid x"); return 1; }
  const unsigned grid = (unsigned)blocks;
  const int rpl = sparse_rpl(R);
  auto go = [&](auto weighted, auto with_fixed) {
    constexpr bool WT = decltype(weighted)::value, FIXED = decltype(with_fixed)::value;
#define NMF_OCD(RPLV) \
  observed_cd_kernel<RPLV, WT, FIXED><<<grid, 256, 0, st>>>(ptr, idx, val, wt, X, F, R, nseg, rbuf, l1, l2, fixed)
    if (rpl <= 1) NMF_OCD(1);
    else if (rpl <= 2) NMF_OCD(2);
    else if (rpl <= 4) NMF_OCD(4);
    else NMF_OCD(8);
#undef NMF_OCD
  };
  if (fixed && wt) go(std::true_type{}, std::true_type{});
  else if (fixed) go(std::false_type{}, std::true_type{});
  else if (wt) go(std::true_type{}, std::false_type{});
  else go(std::false_type{}, std::false_type{});
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace nmfb200
