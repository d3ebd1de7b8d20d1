// Ratio stage of the multiplicative update (nmf.py:78-92) and the small reductions around it.
#include "common.cuh"

namespace nmfb200 {

namespace {

// Where the partials of element idx (of problem b) are: the offset in the first slab, the slab count and stride.  False for
// a padding row of a ragged batch's H, or (LINES) a padding position of a ragged NMFD batch's H lines, which no kernel
// writes.  The kernels below take RAGGED (a.rag set) and LINES (a.line set as well) as template flags, so that their other
// instantiations run the code they always ran.  The ratio-stage kernels take FIXED the same way: `fixed` (R bytes, non-zero
// for a component held at its value, nmfb200_set_fixed_w) predicates the final store of each element on its component.  And
// PEN: `pen` (R floats, the ARD penalties of nmfb200_set_ard) adds pen[r] to the denominator of every element of component r,
// with the fp32 add the scalar l1 takes.
struct PartialAt { int64_t off, stride; int nch; };
template <bool RAGGED, bool LINES = false>
__device__ __forceinline__ bool partial_at(const ApplyArgs& a, int64_t idx, int64_t b, PartialAt& p) {
  if constexpr (RAGGED) {
    const RaggedProblem& rp = a.rag[b];
    const int64_t local = idx - b * a.prob_numel;
    if constexpr (LINES) {                       // NMFD's H: the problem's compact [split][lines][lin] slabs
      const int64_t ln = local / a.line, j = local - ln * a.line;
      if (j >= rp.lin) return false;
      p = PartialAt{rp.part + ln * rp.lin + j, a.prob_numel / a.line * rp.lin, rp.nch[1]};
      return true;
    }
    const int64_t row = local / a.rowlen;
    const int64_t rows = a.rag_launch == kRagW ? a.prob_numel / a.rowlen : rp.rows;
    if (row >= rows) return false;
    p = PartialAt{rp.part + row * a.ldp + (local - row * a.rowlen), rows * a.ldp, rp.nch[a.rag_launch]};
    return true;
  }
  const int64_t row = idx / a.rowlen;
  p = PartialAt{row * a.ldp + (idx - row * a.rowlen), a.chunk_stride, a.nchunks};
  return true;
}

template <bool RAGGED, bool LINES = false, bool FIXED = false, bool PEN = false>
__global__ void __launch_bounds__(256)
apply_update_kernel(ApplyArgs a, const uint8_t* __restrict__ fixed, const float* __restrict__ pen) {
  const int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x;
  float newv = 0.f;
  const int64_t b = a.prob_numel ? idx / a.prob_numel : 0;      // Batch: the element's problem
  PartialAt pa;
  if (idx < a.numel && !batch_skips(a.active, b) && partial_at<RAGGED, LINES>(a, idx, b, pa)) {
    const int64_t off = pa.off;
    const int r = (int)((idx / a.inner) % a.R);
    const float sc = a.out_scale ? *a.out_scale : 1.0f;
    float num = 0.f;
    for (int ch = 0; ch < pa.nch; ++ch) num += a.num[ch * pa.stride + off];
    num *= sc;
    if (a.kappa) num = fmaf(*a.kappa, a.kappa_vec[r], num);
    const float p = a.param[idx];
    float neg = fmaxf(num, 0.f) + kEps;                      // nmf.py:78
    float pos;
    if (a.den) {
      float den = 0.f;
      for (int ch = 0; ch < pa.nch; ++ch) den += a.den[ch * pa.stride + off];
      den *= sc;
      pos = fmaxf(den, 0.f) + kEps;                          // nmf.py:83
    } else {
      pos = a.kl_den[b * a.R + r];                           // nmf.py:368-369 / :381-382 (no relu, no eps)
    }
    if (a.l1 > 0.f) pos += a.l1;                             // nmf.py:85-86
    if constexpr (PEN) pos += pen[r];                        // ARD: l1 of component r
    if (a.l2 > 0.f) pos = fmaf(a.l2, p, pos);                // nmf.py:87-88
    float mult = neg / pos;                                  // nmf.py:89
    if (a.gamma != 1.0f) mult = powf(mult, a.gamma);         // nmf.py:90-91
    newv = p * mult;                                         // nmf.py:92
    if (FIXED && fixed[r]) newv = p;                         // a fixed component keeps its value and still enters absmax
    else a.param[idx] = newv;
  }
  if (a.absmax_bits) {          // one atomic per block: tens of thousands of same-address atomics serialise in L2
    __shared__ float wmax[8];
    float m = newv;
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int i = 1; i < 8; ++i) m = fmaxf(m, wmax[i]);
      if (m > 0.f) atomicMax(a.absmax_bits, __float_as_uint(m));
    }
  }
}

// The ratio stage's inputs without the ratio stage: the summed partials (+ the centring term), nothing clamped.
template <bool RAGGED, bool LINES = false>
__global__ void __launch_bounds__(256)
raw_sum_kernel(ApplyArgs a, float* __restrict__ num_out, float* __restrict__ den_out) {
  const int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int64_t b = a.prob_numel ? idx / a.prob_numel : 0;
  PartialAt pa;
  if (idx >= a.numel || batch_skips(a.active, b) || !partial_at<RAGGED, LINES>(a, idx, b, pa)) return;
  const int64_t off = pa.off;
  const float sc = a.out_scale ? *a.out_scale : 1.0f;
  float num = 0.f;
  for (int ch = 0; ch < pa.nch; ++ch) num += a.num[ch * pa.stride + off];
  num *= sc;
  if (a.kappa) num = fmaf(*a.kappa, a.kappa_vec[(int)((idx / a.inner) % a.R)], num);
  num_out[idx] = num;
  if (den_out) {
    float den = 0.f;
    for (int ch = 0; ch < pa.nch; ++ch) den += a.den[ch * pa.stride + off];
    den_out[idx] = den * sc;
  }
}

// stage 1 for inner == 1: x is (outer, R) row-major; block (b, y) sums a row slab of components [256 y, 256 y + 256).
// Batch: nb blocks per problem along x, each problem's x and partials nprob-strided (outer R and nb R floats).  A ragged
// batch (rag, nprob problems): problem b's own rows, blocks and partials from its plan.
template <bool RAGGED>
__global__ void __launch_bounds__(256)
colsum_rows_kernel(const float* __restrict__ x, int64_t outer, int R, int64_t rows_per_block,
                   float* __restrict__ partial, int64_t nb, const uint8_t* __restrict__ active,
                   const RaggedProblem* __restrict__ rag, int64_t nprob) {
  __shared__ float sh[256];
  int64_t prob, bx;
  if constexpr (RAGGED) {
    prob = ragged_problem(rag, nprob, kRagColsum, blockIdx.x);
    x += prob * outer * R;
    partial += rag[prob].cs_part;
    bx = (int64_t)blockIdx.x - rag[prob].x0[kRagColsum];
    outer = rag[prob].rows;
    rows_per_block = (outer + rag[prob].cs_blocks - 1) / rag[prob].cs_blocks;
  } else {
    prob = (int64_t)blockIdx.x / nb;
    x += prob * outer * R;
    partial += prob * nb * R;
    bx = (int64_t)blockIdx.x - prob * nb;
  }
  if (batch_skips(active, prob)) return;
  const int tid = threadIdx.x;
  const int r0 = blockIdx.y * 256;
  const int Rb = min(R - r0, 256);               // this block's components
  const int ng = 256 / Rb > 0 ? 256 / Rb : 1;    // row groups
  const int g = tid / Rb, r = tid - g * Rb;
  const int64_t row0 = bx * rows_per_block;
  const int64_t row1 = min(outer, row0 + rows_per_block);
  float acc = 0.f;
  if (g < ng)
    for (int64_t row = row0 + g; row < row1; row += ng) acc += x[row * R + r0 + r];
  sh[tid] = acc;
  __syncthreads();
  if (tid < Rb) {
    float t = 0.f;
    for (int k = 0; k < ng; ++k) t += sh[k * Rb + tid];
    partial[bx * R + r0 + tid] = t;
  }
}

// stage 1 for inner > 1: one block per (o, r) run of `inner` contiguous elements.  BATCH: `runs` blocks per problem, problem
// after problem (their runs and partials are contiguous); a problem whose `active` flag is 0 is skipped.
template <bool BATCH = false>
__global__ void __launch_bounds__(256)
colsum_runs_kernel(const float* __restrict__ x, int64_t inner, float* __restrict__ partial, int64_t runs,
                   const uint8_t* __restrict__ active) {
  __shared__ float sh[8];
  if constexpr (BATCH) {
    if (batch_skips(active, (int64_t)blockIdx.x / runs)) return;
  }
  const float* run = x + (int64_t)blockIdx.x * inner;
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < inner; i += 256) acc += run[i];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += sh[k];
    partial[blockIdx.x] = t;      // index o*R + r
  }
}

// stage 1 of a ragged NMFD batch's H: x is nprob problems of (outer, R, inner) activations whose last axis is `line` long,
// one block per (problem, o, r).  Problem b's run (o, r) is the first rag[b].lin positions of each of its inner / line lines,
// summed as colsum_runs_kernel sums a single problem's run of that many elements, its partial at rag[b].cs_part + o R + r.
// A problem whose run is one element (one line, lin 1) is summed as its single fit sums it, by colsum_rows_kernel: block
// (o, r) for o < rag[b].cs_blocks forms that kernel's block-o partial of component r, in its order, in one thread.
__global__ void __launch_bounds__(256)
colsum_lines_kernel(const float* __restrict__ x, int64_t outer, int R, int64_t inner, int64_t line, float* __restrict__ partial,
                    const uint8_t* __restrict__ active, const RaggedProblem* __restrict__ rag) {
  __shared__ float sh[8];
  const int64_t runs = outer * R, prob = (int64_t)blockIdx.x / runs, k = (int64_t)blockIdx.x - prob * runs;
  if (batch_skips(active, prob)) return;
  const RaggedProblem& rp = rag[prob];
  const int64_t lin = rp.lin, n = inner / line * lin;
  x += prob * runs * inner;
  partial += rp.cs_part;
  if (n == 1) {
    const int64_t o = k / R, r = k - o * R;
    if (o >= rp.cs_blocks || threadIdx.x != 0) return;
    const int64_t rpb = (outer + rp.cs_blocks - 1) / rp.cs_blocks, row0 = o * rpb, row1 = min(outer, row0 + rpb);
    const int ng = 256 / R;
    float t = 0.f;
    for (int g = 0; g < ng; ++g) {
      float acc = 0.f;
      for (int64_t row = row0 + g; row < row1; row += ng) acc += x[(row * R + r) * inner];
      t += acc;
    }
    partial[o * R + r] = t;
    return;
  }
  const float* run = x + k * inner;
  float acc = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += 256) {
    const int64_t ln = i / lin;
    acc += run[ln * line + (i - ln * lin)];
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int q = 0; q < 8; ++q) t += sh[q];
    partial[k] = t;
  }
}

// Batch: ceil(R / blockDim) blocks per problem along x; a ragged batch's problem b: its own partials and blocks
template <bool RAGGED>
__global__ void colsum_final_kernel(const float* __restrict__ partial, int64_t nb, int R, float* __restrict__ sums,
                                    const uint8_t* __restrict__ active, const RaggedProblem* __restrict__ rag) {
  const int64_t per = (R + blockDim.x - 1) / blockDim.x;
  const int64_t prob = (int64_t)blockIdx.x / per;
  if (batch_skips(active, prob)) return;
  if constexpr (RAGGED) {
    partial += rag[prob].cs_part;
    nb = rag[prob].cs_blocks;
  } else {
    partial += prob * nb * R;
  }
  sums += prob * R;
  const int r = (int)((int64_t)blockIdx.x - prob * per) * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float t = 0.f;
  for (int64_t b = 0; b < nb; ++b) t += partial[b * R + r];
  sums[r] = t;
}

__device__ __forceinline__ float nan_min(float a, float b) { return (a != a || b != b) ? NAN : fminf(a, b); }
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || b != b) ? NAN : fmaxf(a, b); }

// NaN-sticky min / max so that a NaN in V fails fit()'s non-negativity assertion like torch.all(V >= 0) does
// SEL: the cells where M (contiguous rows x cols: a mask or weights) is 0 are skipped, V is not read there
// Batch: nprob matrices of rows x cols, bstride elements apart (ragged, rag: matrix b's first rag[b].rows rows, or with
// COLS its first rag[b].rows columns)
template <typename TV, typename SEL = NoSel, bool COLS = false>
__global__ void __launch_bounds__(256)
minmax_stage1(const TV* __restrict__ V, int64_t rows, int64_t cols, int64_t ld, float* __restrict__ scratch,
              const SEL* __restrict__ M, int64_t nprob, int64_t bstride, const RaggedProblem* __restrict__ rag) {
  __shared__ float smin[8], smax[8];
  float mn = INFINITY, mx = -INFINITY;
  const int64_t total = nprob * rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (int64_t)gridDim.x * 256) {
    if (!sel_set(M, i)) continue;
    int64_t r = i / cols, c = i - r * cols;
    const int64_t b = nprob > 1 ? r / rows : 0;
    r -= b * rows;
    if (rag && (COLS ? c : r) >= rag[b].rows) continue;
    float v = to_f32(V[b * bstride + r * ld + c]);
    mn = nan_min(mn, v);
    mx = nan_max(mx, v);
  }
  for (int o = 16; o > 0; o >>= 1) {
    mn = nan_min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = nan_max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) { smin[threadIdx.x >> 5] = mn; smax[threadIdx.x >> 5] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) { mn = nan_min(mn, smin[k]); mx = nan_max(mx, smax[k]); }
    scratch[blockIdx.x] = mn;
    scratch[1024 + blockIdx.x] = mx;
  }
}

__global__ void minmax_stage2(const float* __restrict__ scratch, int nb, float* __restrict__ mm) {
  if (threadIdx.x != 0) return;
  float mn = INFINITY, mx = -INFINITY;
  for (int k = 0; k < nb; ++k) { mn = nan_min(mn, scratch[k]); mx = nan_max(mx, scratch[1024 + k]); }
  mm[0] = mn;
  mm[1] = mx;
}

}  // namespace

// Four consecutive elements per thread (same row, same component: inner % 4 == 0), 16-byte loads of the parameter and of every
// partial slab.  Same arithmetic per element as apply_update_kernel.
template <bool RAGGED, bool FIXED = false, bool PEN = false>
__global__ void __launch_bounds__(256)
apply_update_vec4_kernel(ApplyArgs a, const uint8_t* __restrict__ fixed, const float* __restrict__ pen) {
  const int64_t idx = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 4;
  float m = 0.f;
  const int64_t b = a.prob_numel ? idx / a.prob_numel : 0;      // Batch: prob_numel is a multiple of 4 here
  PartialAt pa;      // the four elements share a row; a ragged batch's offsets and strides are multiples of 4 here
  if (idx < a.numel && !batch_skips(a.active, b) && partial_at<RAGGED>(a, idx, b, pa)) {
    const int64_t off = pa.off;
    const int r = (int)((idx / a.inner) % a.R);
    const float sc = a.out_scale ? *a.out_scale : 1.0f;
    float4 num = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int ch = 0; ch < pa.nch; ++ch) {
      const float4 t = *reinterpret_cast<const float4*>(a.num + ch * pa.stride + off);
      num.x += t.x; num.y += t.y; num.z += t.z; num.w += t.w;
    }
    float4 den = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.den) {
      for (int ch = 0; ch < pa.nch; ++ch) {
        const float4 t = *reinterpret_cast<const float4*>(a.den + ch * pa.stride + off);
        den.x += t.x; den.y += t.y; den.z += t.z; den.w += t.w;
      }
    }
    const float klden = a.den ? 0.f : a.kl_den[b * a.R + r];
    float pr = 0.f;
    if constexpr (PEN) pr = pen[r];
    float4 p = *reinterpret_cast<const float4*>(a.param + idx);
    auto one = [&](float pv, float n, float d) {
      n *= sc;
      if (a.kappa) n = fmaf(*a.kappa, a.kappa_vec[r], n);
      const float neg = fmaxf(n, 0.f) + kEps;                  // nmf.py:78
      float pos = a.den ? fmaxf(d * sc, 0.f) + kEps : klden;   // nmf.py:83 / :368-369
      if (a.l1 > 0.f) pos += a.l1;                             // nmf.py:85-86
      if constexpr (PEN) pos += pr;                            // ARD: l1 of component r
      if (a.l2 > 0.f) pos = fmaf(a.l2, pv, pos);               // nmf.py:87-88
      float mult = neg / pos;                                  // nmf.py:89
      if (a.gamma != 1.0f) mult = powf(mult, a.gamma);         // nmf.py:90-91
      return pv * mult;                                        // nmf.py:92
    };
    if (!(FIXED && fixed[r])) {                                // the four elements share component r
      p.x = one(p.x, num.x, den.x); p.y = one(p.y, num.y, den.y); p.z = one(p.z, num.z, den.z); p.w = one(p.w, num.w, den.w);
      *reinterpret_cast<float4*>(a.param + idx) = p;
    }
    m = fmaxf(fmaxf(p.x, p.y), fmaxf(p.z, p.w));
  }
  if (a.absmax_bits) {
    __shared__ float wmax[8];
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int i = 1; i < 8; ++i) m = fmaxf(m, wmax[i]);
      if (m > 0.f) atomicMax(a.absmax_bits, __float_as_uint(m));
    }
  }
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

bool apply_update_vec4_shape(const ApplyArgs& a) {
  return a.inner % 4 == 0 && a.rowlen % 4 == 0 && a.ldp % 4 == 0 && a.numel % 4 == 0 &&
         (a.nchunks == 1 || a.chunk_stride % 4 == 0) && a.prob_numel % 4 == 0 && a.line == 0;
}

int apply_update(const ApplyArgs& a, cudaStream_t st, const uint8_t* fixed, const float* pen) {
  if (a.numel <= 0) return 0;
  if (fixed && (a.rag || a.prob_numel)) { set_error("apply_update: fixed components need a single problem"); return 1; }
  if (pen && (a.rag || a.prob_numel || fixed)) { set_error("apply_update: ARD penalties need a single problem, nothing fixed"); return 1; }
  const bool vec4 = apply_update_vec4_shape(a) && aligned16(a.param) && aligned16(a.num) && (!a.den || aligned16(a.den));
  const unsigned g4 = (unsigned)ceil_div(a.numel / 4, 256), g1 = (unsigned)ceil_div(a.numel, 256);
  if (pen && vec4) apply_update_vec4_kernel<false, false, true><<<g4, 256, 0, st>>>(a, nullptr, pen);
  else if (pen) apply_update_kernel<false, false, false, true><<<g1, 256, 0, st>>>(a, nullptr, pen);
  else if (fixed && vec4) apply_update_vec4_kernel<false, true><<<g4, 256, 0, st>>>(a, fixed, nullptr);
  else if (fixed) apply_update_kernel<false, false, true><<<g1, 256, 0, st>>>(a, fixed, nullptr);
  else if (vec4 && a.rag) apply_update_vec4_kernel<true><<<g4, 256, 0, st>>>(a, nullptr, nullptr);
  else if (vec4) apply_update_vec4_kernel<false><<<g4, 256, 0, st>>>(a, nullptr, nullptr);
  else if (a.rag && a.line) apply_update_kernel<true, true><<<g1, 256, 0, st>>>(a, nullptr, nullptr);
  else if (a.rag) apply_update_kernel<true><<<g1, 256, 0, st>>>(a, nullptr, nullptr);
  else apply_update_kernel<false><<<g1, 256, 0, st>>>(a, nullptr, nullptr);
  NMF_LAUNCH_CHECK();
  return 0;
}

int raw_sum(const ApplyArgs& a, float* num_out, float* den_out, cudaStream_t st) {
  if (a.numel <= 0) return 0;
  const unsigned g1 = (unsigned)ceil_div(a.numel, 256);
  if (a.rag && a.line) raw_sum_kernel<true, true><<<g1, 256, 0, st>>>(a, num_out, a.den ? den_out : nullptr);
  else if (a.rag) raw_sum_kernel<true><<<g1, 256, 0, st>>>(a, num_out, a.den ? den_out : nullptr);
  else raw_sum_kernel<false><<<g1, 256, 0, st>>>(a, num_out, a.den ? den_out : nullptr);
  NMF_LAUNCH_CHECK();
  return 0;
}

static int64_t colsum_blocks(int64_t outer, int64_t inner) {
  if (inner > 1) return outer;   // one per (o, r) run, x R below
  int64_t nb = ceil_div(outer, 64);
  return nb > 1024 ? 1024 : (nb < 1 ? 1 : nb);
}

int64_t colsum_scratch_floats(int64_t outer, int R, int64_t inner) { return colsum_blocks(outer, inner) * R; }

int factor_colsum(const float* x, int64_t outer, int R, int64_t inner, float* scratch, int64_t scratch_floats,
                  float* sums, cudaStream_t st, int64_t nprob, const uint8_t* active, const RaggedProblem* rag,
                  int64_t rag_gx, int64_t rag_line) {
  const int64_t nb = colsum_blocks(outer, inner);
  if (nprob < 1) { set_error("factor_colsum: bad problem count"); return 1; }
  if (rag && rag_line) {   // the scratch was sized where the plans were made (nmfb200_nmfnd_batched_create_ragged)
    if (inner % rag_line || R > 256 || (double)outer * R * nprob > (double)kMaxGridX || ceil_div(R, 64) * nprob > kMaxGridX) {
      set_error("factor_colsum: bad ragged NMFD batch");
      return 1;
    }
    colsum_lines_kernel<<<(unsigned)(outer * R * nprob), 256, 0, st>>>(x, outer, R, inner, rag_line, scratch, active, rag);
    NMF_LAUNCH_CHECK();
    colsum_final_kernel<true><<<(unsigned)(ceil_div(R, 64) * nprob), 64, 0, st>>>(scratch, 0, R, sums, active, rag);
    NMF_LAUNCH_CHECK();
    return 0;
  }
  if (rag) {         // the scratch and grid were checked where the plans were made (nmfb200_nmf_batched_create_ragged)
    if (inner != 1 || rag_gx < 1 || rag_gx > kMaxGridX || R > 256 || nprob > kMaxGridX / 4) {
      set_error("factor_colsum: bad ragged batch");
      return 1;
    }
    colsum_rows_kernel<true><<<(unsigned)rag_gx, 256, 0, st>>>(x, outer, R, 0, scratch, 0, active, rag, nprob);
    NMF_LAUNCH_CHECK();
    colsum_final_kernel<true><<<(unsigned)(ceil_div(R, 64) * nprob), 64, 0, st>>>(scratch, 0, R, sums, active, rag);
    NMF_LAUNCH_CHECK();
    return 0;
  }
  if ((double)nb * R * nprob > (double)scratch_floats) { set_error("factor_colsum: scratch too small"); return 1; }
  if ((double)nb * (inner > 1 ? R : 1) * nprob > (double)kMaxGridX || ceil_div(R, 64) * nprob > kMaxGridX) {
    set_error("factor_colsum: batch passes grid x");
    return 1;
  }
  if (inner > 1) {
    const unsigned gx = (unsigned)(outer * R * nprob);
    if (nprob > 1 || active) colsum_runs_kernel<true><<<gx, 256, 0, st>>>(x, inner, scratch, outer * R, active);
    else colsum_runs_kernel<<<gx, 256, 0, st>>>(x, inner, scratch, outer * R, active);
  } else {
    const int64_t rpb = ceil_div(outer, nb);
    colsum_rows_kernel<false><<<dim3((unsigned)(nb * nprob), (unsigned)ceil_div(R, 256)), 256, 0, st>>>(
        x, outer, R, rpb, scratch, nb, active, nullptr, nprob);
  }
  NMF_LAUNCH_CHECK();
  colsum_final_kernel<false><<<(unsigned)(ceil_div(R, 64) * nprob), 64, 0, st>>>(scratch, nb, R, sums, active, nullptr);
  NMF_LAUNCH_CHECK();
  return 0;
}

int matrix_minmax(const void* V, int vdtype, int64_t rows, int64_t cols, int64_t ld, float* scratch2048, float* mm,
                  cudaStream_t st, CellSel M, int64_t nprob, int64_t bstride, const RaggedProblem* rag, bool rag_cols) {
  if (nprob < 1 || (nprob > 1 && M)) { set_error("matrix_minmax: a batch takes no selector"); return 1; }
  int64_t nb = ceil_div(nprob * rows * cols, 256 * 16);
  if (nb > 1024) nb = 1024;
  if (nb < 1) nb = 1;
  int rc = with_vtype(V, vdtype, [&](auto Vt) {
    using TV = vtype_t<decltype(Vt)>;
    return with_sel(M, [&](auto Mk) {
      if (rag_cols)
        minmax_stage1<TV, sel_t<decltype(Mk)>, true><<<(unsigned)nb, 256, 0, st>>>(Vt, rows, cols, ld, scratch2048, Mk,
                                                                                   nprob, bstride, rag);
      else
        minmax_stage1<TV, sel_t<decltype(Mk)>><<<(unsigned)nb, 256, 0, st>>>(Vt, rows, cols, ld, scratch2048, Mk, nprob,
                                                                            bstride, rag);
      NMF_LAUNCH_CHECK();
      return 0;
    });
  });
  if (rc) return rc;
  minmax_stage2<<<1, 32, 0, st>>>(scratch2048, (int)nb, mm);
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace nmfb200
