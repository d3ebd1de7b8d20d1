// Fused fp32 CUDA-core kernels for one factor update of dense NMF (the exact / any-shape path).
//
// One CTA owns a 64-row block of the "row factor" F and walks 64-column tiles of its column chunk:
//   GEMM-1   S  = F_blk G_tile^T            (registers, 4x4 per thread)        nmf.py:691-693
//   phi      Pn = V * (S+eps)^(beta-2), Pp = (S+eps)^(beta-1)   (in shared)     nmf.py:61-74
//   GEMM-2   num += Pn G_tile, den += Pp G_tile   (registers)                   nmf.py:77,82
// so the (N x C) reconstruction and ratio matrices never exist in global memory.  The H update uses
// (F,G,V) = (H,W,V); the W update uses (W,H,V^T) by reading V through a transposed tile load.
#include "common.cuh"

namespace nmfb200 {

namespace {

constexpr int kTile = 64;   // rows per CTA and columns per tile
constexpr int kLd = 68;     // padded shared-memory pitch (floats): float4-aligned, conflict-free

// 64-column tiles per chunk of the contracted dimension; the last chunks may be short or hold no tile at all
__host__ __device__ inline int64_t chunk_tiles(int64_t Nc, int nchunks) {
  return ((Nc + kTile - 1) / kTile + nchunks - 1) / nchunks;
}

// register blocks of 16 components per thread row of the contraction kernel (Rp = 16 RB >= R)
inline int contract_rb(int R) { return R <= 16 ? 1 : R <= 32 ? 2 : R <= 64 ? 4 : R <= 128 ? 8 : 16; }

template <int MODE>
__device__ __forceinline__ void phi(float v, float s, float bm2, float bm1, float& pn, float& pp) {
  if (MODE == kKL) {
    pn = v / (s + kEps);                 // nmf.py:65
    pp = 0.f;
  } else if (MODE == kEU) {
    pn = v;                              // nmf.py:62-63 (no eps)
    pp = s;
  } else if (MODE == kIS) {
    float r = 1.0f / (s + kEps);         // nmf.py:68-70
    pp = r;
    pn = (r * r) * v;
  } else {
    float x = s + kEps;                  // nmf.py:72-74
    pn = powf(x, bm2) * v;
    pp = powf(x, bm1);
  }
}

template <int RB, bool TRANS, int MODE>
__global__ void __launch_bounds__(256)
simt_contract_kernel(const float* __restrict__ V, int64_t ldv, const float* __restrict__ F,
                     const float* __restrict__ G, int64_t Mr, int64_t Nc, int R, float bm2, float bm1,
                     int nchunks, float* __restrict__ num, float* __restrict__ den, int64_t ldp,
                     int64_t chunk_stride) {
  constexpr int Rp = 16 * RB;
  constexpr bool kTwo = (MODE != kKL);
  extern __shared__ __align__(16) float smem[];
  float* Fs = smem;                 // [Rp][kLd]  Fs[r][row]
  float* Gs = Fs + Rp * kLd;        // [Rp][kLd]  Gs[r][col]
  float* Ps = Gs + Rp * kLd;        // [64][kLd]  V tile, then Pn in place
  float* Qs = Ps + kTile * kLd;     // [64][kLd]  Pp (kTwo only)

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)blockIdx.x * kTile;
  const int chunk = blockIdx.y;
  const int64_t tiles_total = (Nc + kTile - 1) / kTile;
  const int64_t tpc = chunk_tiles(Nc, nchunks);
  const int64_t tile_begin = chunk * tpc;
  const int64_t tile_end = min(tiles_total, tile_begin + tpc);

  for (int idx = tid; idx < kTile * Rp; idx += 256) {
    int row = idx / Rp, r = idx - row * Rp;
    float val = (m0 + row < Mr && r < R) ? F[(m0 + row) * R + r] : 0.f;
    Fs[r * kLd + row] = val;
  }

  float accn[4][RB], accd[4][RB];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int k = 0; k < RB; ++k) { accn[i][k] = 0.f; accd[i][k] = 0.f; }

  for (int64_t tile = tile_begin; tile < tile_end; ++tile) {
    const int64_t c0 = tile * kTile;
    __syncthreads();
    for (int idx = tid; idx < kTile * Rp; idx += 256) {
      int col = idx / Rp, r = idx - col * Rp;
      float val = (c0 + col < Nc && r < R) ? G[(c0 + col) * R + r] : 0.f;
      Gs[r * kLd + col] = val;
    }
    for (int idx = tid; idx < kTile * kTile; idx += 256) {
      int a = idx >> 6, b = idx & 63;
      int row, col;
      float val = 0.f;
      if (!TRANS) {
        row = a; col = b;
        if (m0 + row < Mr && c0 + col < Nc) val = V[(m0 + row) * ldv + c0 + col];
      } else {
        col = a; row = b;
        if (m0 + row < Mr && c0 + col < Nc) val = V[(c0 + col) * ldv + m0 + row];
      }
      Ps[row * kLd + col] = val;
    }
    __syncthreads();

    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 4
    for (int r = 0; r < Rp; ++r) {
      float4 a = *reinterpret_cast<const float4*>(&Fs[r * kLd + 4 * ty]);
      float4 b = *reinterpret_cast<const float4*>(&Gs[r * kLd + 4 * tx]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(av[i], bv[j], s[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float4 v4 = *reinterpret_cast<const float4*>(&Ps[(4 * ty + i) * kLd + 4 * tx]);
      float vv[4] = {v4.x, v4.y, v4.z, v4.w}, pn[4], pp[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) phi<MODE>(vv[j], s[i][j], bm2, bm1, pn[j], pp[j]);
      *reinterpret_cast<float4*>(&Ps[(4 * ty + i) * kLd + 4 * tx]) = make_float4(pn[0], pn[1], pn[2], pn[3]);
      if (kTwo)
        *reinterpret_cast<float4*>(&Qs[(4 * ty + i) * kLd + 4 * tx]) = make_float4(pp[0], pp[1], pp[2], pp[3]);
    }
    __syncthreads();

#pragma unroll 2
    for (int c = 0; c < kTile; c += 4) {
      float4 p[4], q[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        p[i] = *reinterpret_cast<const float4*>(&Ps[(4 * ty + i) * kLd + c]);
        if (kTwo) q[i] = *reinterpret_cast<const float4*>(&Qs[(4 * ty + i) * kLd + c]);
      }
#pragma unroll
      for (int k = 0; k < RB; ++k) {
        float4 g = *reinterpret_cast<const float4*>(&Gs[(tx + 16 * k) * kLd + c]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          accn[i][k] = fmaf(p[i].x, g.x, fmaf(p[i].y, g.y, fmaf(p[i].z, g.z, fmaf(p[i].w, g.w, accn[i][k]))));
          if (kTwo)
            accd[i][k] = fmaf(q[i].x, g.x, fmaf(q[i].y, g.y, fmaf(q[i].z, g.z, fmaf(q[i].w, g.w, accd[i][k]))));
        }
      }
    }
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int64_t row = m0 + 4 * ty + i;
    if (row >= Mr) continue;
#pragma unroll
    for (int k = 0; k < RB; ++k) {
      int r = tx + 16 * k;
      if (r < R) {
        num[chunk * chunk_stride + row * ldp + r] = accn[i][k];
        if (kTwo) den[chunk * chunk_stride + row * ldp + r] = accd[i][k];
      }
    }
  }
}

template <int RB, bool TRANS>
int launch_contract_mode(int mode, dim3 grid, size_t smem, cudaStream_t st, const float* V, int64_t ldv,
                         const float* F, const float* G, int64_t Mr, int64_t Nc, int R, float bm2, float bm1,
                         int nchunks, float* num, float* den, int64_t ldp, int64_t chunk_stride) {
#define NMF_LAUNCH_MODE(M)                                                                              \
  {                                                                                                     \
    auto kern = simt_contract_kernel<RB, TRANS, M>;                                                     \
    NMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    kern<<<grid, 256, smem, st>>>(V, ldv, F, G, Mr, Nc, R, bm2, bm1, nchunks, num, den, ldp,            \
                                  chunk_stride);                                                        \
  }
  switch (mode) {
    case kKL: NMF_LAUNCH_MODE(kKL); break;
    case kEU: NMF_LAUNCH_MODE(kEU); break;
    case kIS: NMF_LAUNCH_MODE(kIS); break;
    default: NMF_LAUNCH_MODE(kGeneric); break;
  }
#undef NMF_LAUNCH_MODE
  NMF_LAUNCH_CHECK();
  return 0;
}

template <int RB>
int launch_contract_rb(int trans, int mode, dim3 grid, cudaStream_t st, const float* V, int64_t ldv,
                       const float* F, const float* G, int64_t Mr, int64_t Nc, int R, float bm2, float bm1,
                       int nchunks, float* num, float* den, int64_t ldp, int64_t chunk_stride) {
  const int Rp = 16 * RB;
  size_t smem = (size_t)(2 * Rp + kTile * (mode == kKL ? 1 : 2)) * kLd * sizeof(float);
  if (trans)
    return launch_contract_mode<RB, true>(mode, grid, smem, st, V, ldv, F, G, Mr, Nc, R, bm2, bm1, nchunks,
                                          num, den, ldp, chunk_stride);
  return launch_contract_mode<RB, false>(mode, grid, smem, st, V, ldv, F, G, Mr, Nc, R, bm2, bm1, nchunks, num,
                                         den, ldp, chunk_stride);
}

// ---- loss ------------------------------------------------------------------------------------

template <int MODE>
__device__ __forceinline__ float loss_term(float v, float s, float beta) {
  if (MODE == kKL) {               // metrics.py:22
    return v * (logf(v + kEps) - logf(s + kEps)) - v + s;
  } else if (MODE == kEU) {        // metrics.py:39
    float d = s - v;
    return 0.5f * d * d;
  } else if (MODE == kIS) {        // metrics.py:56-57
    float te = v + kEps, xe = s + kEps;
    return te / xe - logf(te) + logf(xe) - 1.0f;
  } else {                         // metrics.py:84-96
    float x = s + kEps;
    float t = beta < 0.f ? v + kEps : v;
    float bm = beta - 1.0f;
    return (powf(t, beta) + bm * powf(x, beta) - beta * t * powf(x, bm)) / (beta * bm);
  }
}

__device__ __forceinline__ double block_reduce_sum(double v, double* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) sh[w] = v;
  __syncthreads();
  double t = 0.0;
  if (w == 0) {
    int nw = (blockDim.x + 31) >> 5;
    t = l < nw ? sh[l] : 0.0;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  return t;   // valid in warp 0
}

template <int MODE>
__global__ void __launch_bounds__(256)
simt_loss_kernel(const float* __restrict__ V, int64_t ldv, const float* __restrict__ F,
                 const float* __restrict__ G, int64_t Mr, int64_t Nc, int R, int Rp, float beta, int nchunks,
                 double* __restrict__ block_partials) {
  extern __shared__ __align__(16) float smem[];
  float* Fs = smem;
  float* Gs = Fs + Rp * kLd;
  __shared__ double red[8];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)blockIdx.x * kTile;
  const int chunk = blockIdx.y;
  const int64_t tiles_total = (Nc + kTile - 1) / kTile;
  const int64_t tpc = chunk_tiles(Nc, nchunks);
  const int64_t tile_begin = chunk * tpc;
  const int64_t tile_end = min(tiles_total, tile_begin + tpc);
  for (int idx = tid; idx < kTile * Rp; idx += 256) {
    int row = idx / Rp, r = idx - row * Rp;
    Fs[r * kLd + row] = (m0 + row < Mr && r < R) ? F[(m0 + row) * R + r] : 0.f;
  }
  double acc = 0.0;
  for (int64_t tile = tile_begin; tile < tile_end; ++tile) {
    const int64_t c0 = tile * kTile;
    __syncthreads();
    for (int idx = tid; idx < kTile * Rp; idx += 256) {
      int col = idx / Rp, r = idx - col * Rp;
      Gs[r * kLd + col] = (c0 + col < Nc && r < R) ? G[(c0 + col) * R + r] : 0.f;
    }
    __syncthreads();
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 4
    for (int r = 0; r < Rp; ++r) {
      float4 a = *reinterpret_cast<const float4*>(&Fs[r * kLd + 4 * ty]);
      float4 b = *reinterpret_cast<const float4*>(&Gs[r * kLd + 4 * tx]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(av[i], bv[j], s[i][j]);
    }
    float local = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int64_t row = m0 + 4 * ty + i;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int64_t col = c0 + 4 * tx + j;
        if (row < Mr && col < Nc) local += loss_term<MODE>(V[row * ldv + col], s[i][j], beta);
      }
    }
    acc += (double)local;
  }
  double tot = block_reduce_sum(acc, red);
  if (tid == 0) block_partials[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = tot;
}

__global__ void __launch_bounds__(256) sum_partials_kernel(const double* __restrict__ p, int n, double* out) {
  __shared__ double red[8];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) acc += p[i];
  double tot = block_reduce_sum(acc, red);
  if (threadIdx.x == 0) *out = tot;
}

int loss_chunks(int64_t Mr, int64_t Nc) {
  int64_t rb = ceil_div(Mr, kTile), tiles = ceil_div(Nc, kTile);
  int64_t want = ceil_div(132 * 4, rb);      // a few waves over the 132 SMs of an H100
  if (want < 1) want = 1;
  if (want > tiles) want = tiles;
  return (int)want;
}

}  // namespace

int simt_nmf_max_blocks(int64_t Mr, int64_t Nc) { return (int)(ceil_div(Mr, kTile) * loss_chunks(Mr, Nc)); }

void simt_nmf_plan(int64_t Mr, int64_t Nc, int R, int nchunks, SimtNmfPlan* p) {
  p->rb = contract_rb(R);
  p->tiles_per_chunk = chunk_tiles(Nc, nchunks);
  p->loss_chunks = loss_chunks(Mr, Nc);
  p->loss_tiles_per_chunk = chunk_tiles(Nc, p->loss_chunks);
}

int sum_partials(const double* p, int n, double* out, cudaStream_t st) {
  sum_partials_kernel<<<1, 256, 0, st>>>(p, n, out);
  NMF_LAUNCH_CHECK();
  return 0;
}

int simt_nmf_contract(const float* V, int64_t ldv, int trans, const float* F, const float* G, int64_t Mr,
                      int64_t Nc, int R, double beta, int nchunks, float* num, float* den, int64_t ldp,
                      int64_t chunk_stride, cudaStream_t st) {
  if (R < 1 || R > 256) { set_error("simt_nmf_contract: rank must be in [1, 256]"); return 1; }
  int mode = beta_mode(beta);
  float bm2 = (float)(beta - 2.0), bm1 = (float)(beta - 1.0);
  dim3 grid((unsigned)ceil_div(Mr, kTile), (unsigned)nchunks);
#define NMF_RB(RBV)                                                                                       \
  return launch_contract_rb<RBV>(trans, mode, grid, st, V, ldv, F, G, Mr, Nc, R, bm2, bm1, nchunks, num, den, \
                                 ldp, chunk_stride)
  switch (contract_rb(R)) {
    case 1: NMF_RB(1);
    case 2: NMF_RB(2);
    case 4: NMF_RB(4);
    case 8: NMF_RB(8);
    default: NMF_RB(16);
  }
#undef NMF_RB
}

int simt_nmf_loss(const float* V, int64_t ldv, const float* F, const float* G, int64_t Mr, int64_t Nc, int R,
                  double beta, double* block_partials, int max_blocks, double* loss_dev, cudaStream_t st) {
  if (R < 1 || R > 256) { set_error("simt_nmf_loss: rank must be in [1, 256]"); return 1; }
  int nchunks = loss_chunks(Mr, Nc);
  dim3 grid((unsigned)ceil_div(Mr, kTile), (unsigned)nchunks);
  int nblocks = (int)(grid.x * grid.y);
  if (nblocks > max_blocks) { set_error("simt_nmf_loss: partial buffer too small"); return 1; }
  int Rp = (int)round_up(R, 16);
  size_t smem = (size_t)2 * Rp * kLd * sizeof(float);
  int mode = beta_mode(beta);
#define NMF_LOSS(M)                                                                                     \
  {                                                                                                     \
    auto kern = simt_loss_kernel<M>;                                                                    \
    NMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    kern<<<grid, 256, smem, st>>>(V, ldv, F, G, Mr, Nc, R, Rp, (float)beta, nchunks, block_partials);   \
  }
  switch (mode) {
    case kKL: NMF_LOSS(kKL); break;
    case kEU: NMF_LOSS(kEU); break;
    case kIS: NMF_LOSS(kIS); break;
    default: NMF_LOSS(kGeneric); break;
  }
#undef NMF_LOSS
  NMF_LAUNCH_CHECK();
  return sum_partials(block_partials, nblocks, loss_dev, st);
}

}  // namespace nmfb200
