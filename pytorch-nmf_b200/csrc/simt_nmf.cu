// Fused fp32 CUDA-core kernels for one factor update of dense NMF (the exact / any-shape path).
//
// One CTA owns a 64-row block of the "row factor" F and walks 64-column tiles of its column chunk:
//   GEMM-1   S  = F_blk G_tile^T            (registers, 4x4 per thread)        nmf.py:691-693
//   phi      Pn = V * (S+eps)^(beta-2), Pp = (S+eps)^(beta-1)   (in shared)     nmf.py:61-74
//   GEMM-2   num += Pn G_tile, den += Pp G_tile   (registers)                   nmf.py:77,82
// so the (N x C) reconstruction and ratio matrices never exist in global memory.  The H update uses
// (F,G,V) = (H,W,V); the W update uses (W,H,V^T) by reading V through a transposed tile load.
//
// Ranks above 256 (RB = 16, Rp = 256): S sums over rank chunks of 256 components staged one after another through the same
// Fs / Gs buffers, and each CTA accumulates num / den for one output block of 256 components (blockIdx.z).  Its own chunk
// runs last, so its G slice is still in Gs for GEMM-2.  S is recomputed once per output block: with nb = ceil(R / 256)
// blocks the contraction does (nb + 1) / 2 (KL) or (nb + 2) / 3 (two outputs) times the minimal FLOPs.  With one block
// (R <= 256) the kernel is the single-chunk kernel it always was: grid z = 1, F loaded once per CTA.
//
// SEL (common.cuh), a fit on the observed cells of V only: the kernel loads the uint8 mask tile beside the V tile, through the
// same (possibly transposed) tile load, reads V only where the mask is set, and selects pn = pp = 0 at the missing cells.  It
// always forms both outputs: at beta 1 pp is the mask itself (den = M G, not the column sums of G).  A weighted fit loads the
// fp32 weight tile the same way, reads V only where the weight is non-zero, and multiplies where the mask selects: pn *= w,
// pp *= w, and pp = w at beta 1.  The unmasked instantiations (NoSel) take no branch on it.
//
// Batch (common.cuh, batched NMF): grid x holds the row blocks of every problem, problem after problem; a CTA reads its
// problem's V, F and G and writes its partials at the problem's offsets, and otherwise runs the single problem's plan and
// arithmetic unchanged, so each problem's partials equal a single-problem launch's bit for bit.  In a ragged batch
// (Batch::rag) each problem's plan is that of its own row count: a CTA finds its problem by a binary search over the
// problems' first blocks on grid x, which holds every problem's (chunk, row block) pairs; it reads no row past the problem's.
//
// kVFree (sparse targets at beta != 1, 2): the contraction forms only den += (S+eps)^(beta-1) G_tile and reads no V, with
// kGeneric's plan, staging and arithmetic, so its den partials equal kGeneric's bit for bit whatever V holds; the loss sums
// (S+eps)^beta over every cell, again without V.
//
// kPlcaFill (common.cuh; a masked PLCA fit, fp32 V and the uint8 mask only): the masked KL numerator pn = v / (s+eps) at the
// observed cells, and pp = s / (s+eps) at the missing ones -- the expected complete data of the EM there -- in place of the
// mask.  The CTAs of output block 0 also sum s over their observed cells (fp32 per tile and thread, double across tiles,
// then one fixed-order block reduction) into one partial each, so q_O comes out of the same pass.
//
// kNumOnly (the coordinate-descent solver, cd.cu): the contraction forms only num += V_tile G_tile, with kEU's plan, staging
// and loop order, and skips GEMM-1 and phi -- at beta 2 phi leaves the V tile as it is -- so its num partials equal kEU's bit
// for bit.  It stages no F (Gs starts the shared memory), and runs without a selector, up to rank 256: one problem, or a
// batch (BATCH) in which every problem runs the single problem's plan.
#include "common.cuh"

namespace nmfb200 {

namespace {

constexpr int kTile = 64;   // rows per CTA and columns per tile
constexpr int kVFree = 4;   // MODE of the V-free kernels, beside BetaMode's kKL ... kGeneric
constexpr int kNumOnly = 6; // MODE of the numerator-only kernels (common.cuh's kPlcaFill is 5)
constexpr int kLd = 68;     // padded shared-memory pitch (floats): float4-aligned, conflict-free

// 64-column tiles per chunk of the contracted dimension; the last chunks may be short or hold no tile at all
__host__ __device__ inline int64_t chunk_tiles(int64_t Nc, int nchunks) {
  return ((Nc + kTile - 1) / kTile + nchunks - 1) / nchunks;
}

// register blocks of 16 components per thread row of the contraction kernel (Rp = 16 RB >= R)
inline int contract_rb(int R) { return R <= 16 ? 1 : R <= 32 ? 2 : R <= 64 ? 4 : R <= 128 ? 8 : 16; }

// GEMM-1 over `klen` components of the staged chunk: s[i][j] += Fs[r][4 ty + i] Gs[r][4 tx + j], r ascending
__device__ __forceinline__ void gemm1(const float* Fs, const float* Gs, int klen, int tx, int ty, float (&s)[4][4]) {
#pragma unroll 4
  for (int r = 0; r < klen; ++r) {
    float4 a = *reinterpret_cast<const float4*>(&Fs[r * kLd + 4 * ty]);
    float4 b = *reinterpret_cast<const float4*>(&Gs[r * kLd + 4 * tx]);
    float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = fmaf(av[i], bv[j], s[i][j]);
  }
}

// components [k0, k0 + Rp) of `rows` consecutive rows of X (R columns) from row x0, transposed into Xs[r][row] (zero outside)
__device__ __forceinline__ void stage_chunk(float* Xs, const float* __restrict__ X, int64_t x0, int64_t nx, int R, int k0,
                                            int Rp, int tid) {
  for (int idx = tid; idx < kTile * Rp; idx += 256) {
    int row = idx / Rp, r = idx - row * Rp;
    Xs[r * kLd + row] = (x0 + row < nx && k0 + r < R) ? X[(x0 + row) * R + k0 + r] : 0.f;
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

template <int RB, bool TRANS, int MODE, typename TV, typename SEL = NoSel, bool BATCH = false, bool RAGGED = false>
__global__ void __launch_bounds__(256)
simt_contract_kernel(const TV* __restrict__ V, int64_t ldv, const float* __restrict__ F,
                     const float* __restrict__ G, int64_t Mr, int64_t Nc, int R, float bm2, float bm1,
                     int nchunks, float* __restrict__ num, float* __restrict__ den, int64_t ldp,
                     int64_t chunk_stride, const SEL* __restrict__ Mk, int64_t ldm, Batch bt,
                     double* __restrict__ qobs_part) {
  constexpr bool MASK = !std::is_same<SEL, NoSel>::value;
  constexpr bool WEIGHT = kWeighted<SEL>;
  constexpr bool kFill = (MODE == kPlcaFill);
  static_assert(!kFill || (std::is_same<SEL, uint8_t>::value && std::is_same<TV, float>::value && !BATCH),
                "kPlcaFill: fp32 V, the uint8 mask, one problem");
  constexpr int Rp = 16 * RB;
  constexpr bool kDenOnly = (MODE == kVFree);
  constexpr bool kNumOnly_ = (MODE == kNumOnly);
  static_assert(!kNumOnly_ || !MASK, "kNumOnly: no selector");
  constexpr bool kNum = !kDenOnly;
  constexpr bool kTwo = !kNumOnly_ && ((MODE != kKL) || MASK);
  extern __shared__ __align__(16) float smem[];
  float* Fs = smem;                 // [Rp][kLd]  Fs[r][row] (kNumOnly: none)
  float* Gs = Fs + (kNumOnly_ ? 0 : Rp * kLd);     // [Rp][kLd]  Gs[r][col]
  float* Ps = Gs + Rp * kLd;        // [64][kLd]  V tile, then Pn in place
  float* Qs = kDenOnly ? Ps : Ps + kTile * kLd;     // [64][kLd]  Pp (kTwo only; kVFree: in Ps's place); MASK: the selector first

  // BATCH (NoSel only): this block's problem and its row block within it; the problem's pointers.  The single-problem
  // instantiations compile none of it.  RAGGED (a ragged batch, bt.rag) also takes the problem's rows (F's for the H update,
  // the contracted ones for the W update), chunks and partial slabs from its plan, and its chunk from grid x; the uniform
  // batch instantiations compile none of that.
  static_assert(!RAGGED || (BATCH && !kNumOnly_), "RAGGED: a batch of MU contractions");
  int64_t bx = blockIdx.x;
  int chunk = blockIdx.y;
  if constexpr (RAGGED) {
    const int64_t prob = ragged_problem(bt.rag, bt.n, bt.rag_launch, bx);
    if (batch_skips(bt.active, prob)) return;
    const RaggedProblem& p = bt.rag[prob];
    if (bt.rag_launch == kRagW) Nc = p.rows;
    else Mr = p.rows;
    nchunks = p.nch[bt.rag_launch];
    const int64_t nbx = (Mr + kTile - 1) / kTile;
    bx -= p.x0[bt.rag_launch];
    chunk = (int)(bx / nbx);
    bx -= chunk * nbx;
    chunk_stride = Mr * ldp;
    V += prob * bt.v; F += prob * bt.f; G += prob * bt.g;
    if (kNum) num += p.part;
    if (kTwo) den += p.part;
  } else if constexpr (BATCH) {
    const int64_t nbx = (Mr + kTile - 1) / kTile;
    const int64_t prob = bx / nbx;
    if (batch_skips(bt.active, prob)) return;
    bx -= prob * nbx;
    V += prob * bt.v; F += prob * bt.f; G += prob * bt.g;
    if (kNum) num += prob * bt.p;
    if (kTwo) den += prob * bt.p;
  }

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = bx * kTile;
  const int64_t tiles_total = (Nc + kTile - 1) / kTile;
  const int64_t tpc = chunk_tiles(Nc, nchunks);
  const int64_t tile_begin = chunk * tpc;
  const int64_t tile_end = min(tiles_total, tile_begin + tpc);
  // rank blocks (R > 256 only: RB = 16): nb chunks of S's sum, this CTA's output block ob
  const int nb = RB == 16 ? (int)gridDim.z : 1;
  const int ob = RB == 16 ? (int)blockIdx.z : 0;
  const bool multi = nb > 1;

  if (!multi && !kNumOnly_) stage_chunk(Fs, F, m0, Mr, R, 0, Rp, tid);

  float accn[4][RB], accd[4][RB];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int k = 0; k < RB; ++k) { accn[i][k] = 0.f; accd[i][k] = 0.f; }
  double qacc = 0.0;                // kFill: this thread's sum of s over its observed cells

  for (int64_t tile = tile_begin; tile < tile_end; ++tile) {
    const int64_t c0 = tile * kTile;
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
    for (int t = 0; t < nb; ++t) {
      const int k0 = multi ? (ob + 1 + t) % nb * Rp : 0;     // the own block last: its G slice stays in Gs for GEMM-2
      __syncthreads();
      if (multi) stage_chunk(Fs, F, m0, Mr, R, k0, Rp, tid);
      stage_chunk(Gs, G, c0, Nc, R, k0, Rp, tid);
      if (kNum && t == 0) {
        for (int idx = tid; idx < kTile * kTile; idx += 256) {
          int a = idx >> 6, b = idx & 63;
          int row, col;
          float val = 0.f;
          if (!TRANS) {
            row = a; col = b;
          } else {
            col = a; row = b;
          }
          const bool in = m0 + row < Mr && c0 + col < Nc;
          if constexpr (!MASK) {
            if (in) val = to_f32(TRANS ? V[(c0 + col) * ldv + m0 + row] : V[(m0 + row) * ldv + c0 + col]);
          } else if constexpr (WEIGHT) {
            const float w = in ? (TRANS ? Mk[(c0 + col) * ldm + m0 + row] : Mk[(m0 + row) * ldm + c0 + col]) : 0.f;
            if (w != 0.f) val = to_f32(TRANS ? V[(c0 + col) * ldv + m0 + row] : V[(m0 + row) * ldv + c0 + col]);
            Qs[row * kLd + col] = w;
          } else {
            const bool seen = in && (TRANS ? Mk[(c0 + col) * ldm + m0 + row] : Mk[(m0 + row) * ldm + c0 + col]) != 0;
            if (seen) val = to_f32(TRANS ? V[(c0 + col) * ldv + m0 + row] : V[(m0 + row) * ldv + c0 + col]);
            Qs[row * kLd + col] = seen ? 1.f : 0.f;
          }
          Ps[row * kLd + col] = val;
        }
      }
      __syncthreads();
      if (kNumOnly_) continue;
      if (multi)
        gemm1(Fs, Gs, min(Rp, (R - k0 + 15) & ~15), tx, ty, s);   // the chunk's components, zero-padded to 16
      else
        gemm1(Fs, Gs, Rp, tx, ty, s);
    }
    float qloc = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (kNumOnly_) continue;         // num = V G: the V tile is GEMM-2's operand as it stands
      if (kDenOnly) {
        float pp[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float x = s[i][j] + kEps;        // phi<kGeneric>'s pp
          pp[j] = powf(x, bm1);
        }
        *reinterpret_cast<float4*>(&Qs[(4 * ty + i) * kLd + 4 * tx]) = make_float4(pp[0], pp[1], pp[2], pp[3]);
        continue;
      }
      float4 v4 = *reinterpret_cast<const float4*>(&Ps[(4 * ty + i) * kLd + 4 * tx]);
      float vv[4] = {v4.x, v4.y, v4.z, v4.w}, pn[4], pp[4];
      if constexpr (!kFill) {
#pragma unroll
        for (int j = 0; j < 4; ++j) phi<MODE>(vv[j], s[i][j], bm2, bm1, pn[j], pp[j]);
      }
      if (MASK) {
        float4 m4 = *reinterpret_cast<const float4*>(&Qs[(4 * ty + i) * kLd + 4 * tx]);
        const float mv[4] = {m4.x, m4.y, m4.z, m4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const bool seen = mv[j] != 0.f;
          if constexpr (WEIGHT) {
            pn[j] = seen ? pn[j] * mv[j] : 0.f;
            pp[j] = MODE == kKL ? mv[j] : (seen ? pp[j] * mv[j] : 0.f);
          } else if constexpr (kFill) {
            // one division per cell: v / (s+eps) where observed (kKL's pn), s / (s+eps) where missing
            const float r = (seen ? vv[j] : s[i][j]) / (s[i][j] + kEps);
            pn[j] = seen ? r : 0.f;
            pp[j] = seen ? 0.f : r;
            if (seen) qloc += s[i][j];
          } else {
            pn[j] = seen ? pn[j] : 0.f;
            pp[j] = MODE == kKL ? mv[j] : (seen ? pp[j] : 0.f);
          }
        }
      }
      *reinterpret_cast<float4*>(&Ps[(4 * ty + i) * kLd + 4 * tx]) = make_float4(pn[0], pn[1], pn[2], pn[3]);
      if (kTwo)
        *reinterpret_cast<float4*>(&Qs[(4 * ty + i) * kLd + 4 * tx]) = make_float4(pp[0], pp[1], pp[2], pp[3]);
    }
    if (kFill) qacc += (double)qloc;
    __syncthreads();

#pragma unroll 2
    for (int c = 0; c < kTile; c += 4) {
      float4 p[4], q[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (kNum) p[i] = *reinterpret_cast<const float4*>(&Ps[(4 * ty + i) * kLd + c]);
        if (kTwo) q[i] = *reinterpret_cast<const float4*>(&Qs[(4 * ty + i) * kLd + c]);
      }
#pragma unroll
      for (int k = 0; k < RB; ++k) {
        float4 g = *reinterpret_cast<const float4*>(&Gs[(tx + 16 * k) * kLd + c]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (kNum)
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
      int r = ob * Rp + tx + 16 * k;
      if (r < R) {
        if (kNum) num[chunk * chunk_stride + row * ldp + r] = accn[i][k];
        if (kTwo) den[chunk * chunk_stride + row * ldp + r] = accd[i][k];
      }
    }
  }
  if constexpr (kFill) {
    // every cell's s is the same in each output block: block 0 alone counts it.  (The row loop above exits no thread.)
    if (qobs_part && ob == 0) {
      __shared__ double red[8];
      const double tot = block_reduce_sum(qacc, red);
      if (tid == 0) qobs_part[(int64_t)chunk * gridDim.x + blockIdx.x] = tot;
    }
  }
}

template <int RB, bool TRANS, typename TV, typename SEL, bool BATCH, bool RAGGED = false>
int launch_contract_mode(int mode, dim3 grid, size_t smem, cudaStream_t st, const TV* V, int64_t ldv,
                         const float* F, const float* G, int64_t Mr, int64_t Nc, int R, float bm2, float bm1,
                         int nchunks, float* num, float* den, int64_t ldp, int64_t chunk_stride, const SEL* Mk,
                         int64_t ldm, const Batch& bt) {
#define NMF_LAUNCH_MODE(M)                                                                              \
  {                                                                                                     \
    auto kern = simt_contract_kernel<RB, TRANS, M, TV, SEL, BATCH, RAGGED>;                             \
    NMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    kern<<<grid, 256, smem, st>>>(V, ldv, F, G, Mr, Nc, R, bm2, bm1, nchunks, num, den, ldp,            \
                                  chunk_stride, Mk, ldm, bt, nullptr);                                  \
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

template <int RB, typename TV, typename SEL>
int launch_contract_rb(int trans, int mode, dim3 grid, cudaStream_t st, const TV* V, int64_t ldv,
                       const float* F, const float* G, int64_t Mr, int64_t Nc, int R, float bm2, float bm1,
                       int nchunks, float* num, float* den, int64_t ldp, int64_t chunk_stride, const SEL* Mk,
                       int64_t ldm, const Batch& bt) {
  const int Rp = 16 * RB;
  constexpr bool MASK = !std::is_same<SEL, NoSel>::value;
  size_t smem = (size_t)(2 * Rp + kTile * (mode == kKL && !MASK ? 1 : 2)) * kLd * sizeof(float);
  // a batch runs the BATCH instantiations (no selector), a ragged one the RAGGED ones; one problem the single-problem ones
  if constexpr (std::is_same<SEL, NoSel>::value) {
    if (bt.rag) {
      if (trans)
        return launch_contract_mode<RB, true, TV, SEL, true, true>(mode, grid, smem, st, V, ldv, F, G, Mr, Nc, R, bm2, bm1,
                                                                   nchunks, num, den, ldp, chunk_stride, Mk, ldm, bt);
      return launch_contract_mode<RB, false, TV, SEL, true, true>(mode, grid, smem, st, V, ldv, F, G, Mr, Nc, R, bm2, bm1,
                                                                  nchunks, num, den, ldp, chunk_stride, Mk, ldm, bt);
    }
    if (bt.n > 1 || bt.active) {
      if (trans)
        return launch_contract_mode<RB, true, TV, SEL, true>(mode, grid, smem, st, V, ldv, F, G, Mr, Nc, R, bm2, bm1,
                                                             nchunks, num, den, ldp, chunk_stride, Mk, ldm, bt);
      return launch_contract_mode<RB, false, TV, SEL, true>(mode, grid, smem, st, V, ldv, F, G, Mr, Nc, R, bm2, bm1,
                                                            nchunks, num, den, ldp, chunk_stride, Mk, ldm, bt);
    }
  }
  if (trans)
    return launch_contract_mode<RB, true, TV, SEL, false>(mode, grid, smem, st, V, ldv, F, G, Mr, Nc, R, bm2, bm1, nchunks,
                                                          num, den, ldp, chunk_stride, Mk, ldm, bt);
  return launch_contract_mode<RB, false, TV, SEL, false>(mode, grid, smem, st, V, ldv, F, G, Mr, Nc, R, bm2, bm1, nchunks,
                                                         num, den, ldp, chunk_stride, Mk, ldm, bt);
}

// ---- loss ------------------------------------------------------------------------------------

// SEL: the sum runs over the observed cells only (the missing ones are dropped, not zeroed: at beta != 0, 1, 2 a zeroed
// cell would still add eps^beta / beta); a weighted fit adds w * term over the cells with w != 0
template <int MODE, typename TV, typename SEL = NoSel, bool BATCH = false, bool RAGGED = false>
__global__ void __launch_bounds__(256)
simt_loss_kernel(const TV* __restrict__ V, int64_t ldv, const float* __restrict__ F,
                 const float* __restrict__ G, int64_t Mr, int64_t Nc, int R, int Rp, float beta, int nchunks,
                 double* __restrict__ block_partials, const SEL* __restrict__ Mk, int64_t ldm, Batch bt) {
  extern __shared__ __align__(16) float smem[];
  float* Fs = smem;
  float* Gs = Fs + Rp * kLd;
  __shared__ double red[8];
  // BATCH (NoSel only): problem `prob`'s blocks write its own run of gridDim.y x nbx partials, laid out as a single
  // problem's.  RAGGED (a ragged batch, bt.rag): the problem's rows and loss chunks from its plan, its chunk from grid x,
  // its run of partials at its loss_part.
  static_assert(!RAGGED || BATCH, "RAGGED: a batch");
  int64_t bx = blockIdx.x, part = 0;
  int chunk = blockIdx.y;
  float sc = 1.f;                    // BATCH, KL: the problem's bt.scale
  if constexpr (RAGGED) {
    const int64_t prob = ragged_problem(bt.rag, bt.n, kRagLoss, bx);
    if (batch_skips(bt.active, prob)) return;
    const RaggedProblem& p = bt.rag[prob];
    Mr = p.rows;
    nchunks = p.loss_chunks;
    const int64_t nbx = (Mr + kTile - 1) / kTile;
    bx -= p.x0[kRagLoss];
    part = p.loss_part + bx;
    chunk = (int)(bx / nbx);
    bx -= chunk * nbx;
    V += prob * bt.v; F += prob * bt.f; G += prob * bt.g;
    if (MODE == kKL && bt.scale) sc = bt.scale[prob];
  } else if constexpr (BATCH) {
    const int64_t nbx = (Mr + kTile - 1) / kTile;
    const int64_t prob = bx / nbx;
    if (batch_skips(bt.active, prob)) return;
    bx -= prob * nbx;
    part = (prob * gridDim.y + blockIdx.y) * nbx + bx;
    V += prob * bt.v; F += prob * bt.f; G += prob * bt.g;
    if (MODE == kKL && bt.scale) sc = bt.scale[prob];
  }
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = bx * kTile;
  const int64_t tiles_total = (Nc + kTile - 1) / kTile;
  const int64_t tpc = chunk_tiles(Nc, nchunks);
  const int64_t tile_begin = chunk * tpc;
  const int64_t tile_end = min(tiles_total, tile_begin + tpc);
  // Rp: the staged chunk width, round_up(R, 16) up to 256; above that S sums over rank chunks of 256 (F re-staged per chunk)
  const bool multi = R > Rp;
  if (!multi) stage_chunk(Fs, F, m0, Mr, R, 0, Rp, tid);
  double acc = 0.0;
  for (int64_t tile = tile_begin; tile < tile_end; ++tile) {
    const int64_t c0 = tile * kTile;
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
    for (int k0 = 0; k0 < R; k0 += Rp) {
      __syncthreads();
      if (multi) stage_chunk(Fs, F, m0, Mr, R, k0, Rp, tid);
      stage_chunk(Gs, G, c0, Nc, R, k0, Rp, tid);
      __syncthreads();
      gemm1(Fs, Gs, min(Rp, (R - k0 + 15) & ~15), tx, ty, s);
    }
    float local = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int64_t row = m0 + 4 * ty + i;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int64_t col = c0 + 4 * tx + j;
        if constexpr (kWeighted<SEL>) {
          const float w = row < Mr && col < Nc ? Mk[row * ldm + col] : 0.f;
          if (w != 0.f) local += loss_term_w<MODE>(to_f32(V[row * ldv + col]), s[i][j], beta, w);
        } else if (row < Mr && col < Nc && sel_set(Mk, row * ldm + col)) {
          if (MODE == kVFree) local += powf(s[i][j] + kEps, beta);       // nmf.py:635-636, before the division by beta
          else if (BATCH && MODE == kKL) local += loss_term<MODE>(sc * to_f32(V[row * ldv + col]), sc * s[i][j], beta);
          else local += loss_term<MODE>(to_f32(V[row * ldv + col]), s[i][j], beta);
        }
      }
    }
    acc += (double)local;
  }
  double tot = block_reduce_sum(acc, red);
  if (tid == 0) block_partials[BATCH ? part : (int64_t)blockIdx.y * gridDim.x + blockIdx.x] = tot;
}

// one block per problem (grid x): out[b] = the sum of p[b n, (b + 1) n); RAGGED: of problem b's own loss partials
template <bool RAGGED>
__global__ void __launch_bounds__(256) sum_partials_kernel(const double* __restrict__ p, int n, double* out,
                                                           const uint8_t* __restrict__ active,
                                                           const RaggedProblem* __restrict__ rag) {
  __shared__ double red[8];
  const int64_t b = blockIdx.x;
  if (batch_skips(active, b)) return;
  if constexpr (RAGGED) {
    p += rag[b].loss_part;
    n = (int)rag[b].loss_n;
  } else {
    p += b * n;
  }
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) acc += p[i];
  double tot = block_reduce_sum(acc, red);
  if (threadIdx.x == 0) out[b] = tot;
}

int loss_chunks(int64_t Mr, int64_t Nc) {
  int64_t rb = ceil_div(Mr, kTile), tiles = ceil_div(Nc, kTile);
  int64_t want = ceil_div(132 * 4, rb);      // a few waves over the 132 SMs of an H100
  if (want < 1) want = 1;
  if (want > tiles) want = tiles;
  return (int)want;
}

}  // namespace

int simt_rank_blocks(int R) { return (int)ceil_div(R, 256); }

int simt_nmf_max_blocks(int64_t Mr, int64_t Nc) { return (int)(ceil_div(Mr, kTile) * loss_chunks(Mr, Nc)); }

void simt_nmf_plan(int64_t Mr, int64_t Nc, int R, int nchunks, SimtNmfPlan* p) {
  p->rb = contract_rb(R);
  p->tiles_per_chunk = chunk_tiles(Nc, nchunks);
  p->loss_chunks = loss_chunks(Mr, Nc);
  p->loss_tiles_per_chunk = chunk_tiles(Nc, p->loss_chunks);
}

int sum_partials(const double* p, int n, double* out, cudaStream_t st, int64_t nprob, const uint8_t* active,
                 const RaggedProblem* rag) {
  if (nprob < 1 || nprob > kMaxGridX) { set_error("sum_partials: bad problem count"); return 1; }
  if (rag) sum_partials_kernel<true><<<(unsigned)nprob, 256, 0, st>>>(p, n, out, active, rag);
  else sum_partials_kernel<false><<<(unsigned)nprob, 256, 0, st>>>(p, n, out, active, nullptr);
  NMF_LAUNCH_CHECK();
  return 0;
}

// grid x of a batched launch: nbx blocks per problem for bt.n problems; a ragged batch's own sum of blocks
static int batch_grid_x(int64_t nbx, const Batch& bt, const char* who, unsigned* x) {
  if (bt.rag) {
    if (bt.rag_gx < 1 || bt.rag_gx > kMaxGridX) { set_error(std::string(who) + ": ragged blocks pass grid x"); return 1; }
    *x = (unsigned)bt.rag_gx;
    return 0;
  }
  if (bt.n < 1 || nbx > kMaxGridX / bt.n) { set_error(std::string(who) + ": batch x row blocks pass grid x"); return 1; }
  *x = (unsigned)(nbx * bt.n);
  return 0;
}

int simt_nmf_contract(const void* V, int vdtype, int64_t ldv, int trans, const float* F, const float* G, int64_t Mr,
                      int64_t Nc, int R, double beta, int nchunks, float* num, float* den, int64_t ldp,
                      int64_t chunk_stride, CellSel M, int64_t ldm, cudaStream_t st, const Batch& bt) {
  if (R < 1) { set_error("simt_nmf_contract: rank must be positive"); return 1; }
  if (bt.n > 1 && M) { set_error("simt_nmf_contract: a batch takes no selector"); return 1; }
  int mode = beta_mode(beta);
  float bm2 = (float)(beta - 2.0), bm1 = (float)(beta - 1.0);
  unsigned gx;
  if (batch_grid_x(ceil_div(Mr, kTile), bt, "simt_nmf_contract", &gx)) return 1;
  if (bt.rag && R > 256) { set_error("simt_nmf_contract: a ragged batch takes rank <= 256"); return 1; }
  dim3 grid(gx, bt.rag ? 1u : (unsigned)nchunks, (unsigned)simt_rank_blocks(R));     // ragged: the chunks are on grid x
  const int rb = contract_rb(R);
  return with_vtype(V, vdtype, [&](auto Vt) {
    using TV = vtype_t<decltype(Vt)>;
    return with_sel(M, [&](auto Mk) {
      using SEL = sel_t<decltype(Mk)>;
#define NMF_RB(RBV)                                                                                                     \
  return launch_contract_rb<RBV, TV, SEL>(trans, mode, grid, st, Vt, ldv, F, G, Mr, Nc, R, bm2, bm1, nchunks, num, den, \
                                          ldp, chunk_stride, Mk, M ? ldm : 0, bt)
      switch (rb) {
        case 1: NMF_RB(1);
        case 2: NMF_RB(2);
        case 4: NMF_RB(4);
        case 8: NMF_RB(8);
        default: NMF_RB(16);
      }
#undef NMF_RB
    });
  });
}

int simt_nmf_loss(const void* V, int vdtype, int64_t ldv, const float* F, const float* G, int64_t Mr, int64_t Nc, int R,
                  double beta, double* block_partials, int max_blocks, double* loss_dev, CellSel M, int64_t ldm,
                  cudaStream_t st, const Batch& bt) {
  if (R < 1) { set_error("simt_nmf_loss: rank must be positive"); return 1; }
  if (bt.n > 1 && M) { set_error("simt_nmf_loss: a batch takes no selector"); return 1; }
  int nchunks = loss_chunks(Mr, Nc);
  unsigned gx;
  if (batch_grid_x(ceil_div(Mr, kTile), bt, "simt_nmf_loss", &gx)) return 1;
  dim3 grid(gx, bt.rag ? 1u : (unsigned)nchunks);                    // ragged: the chunks are on grid x
  const int nblocks = (int)(ceil_div(Mr, kTile) * nchunks);          // per problem (ragged: every problem's, below)
  const double total = bt.rag ? (double)bt.rag_gx : (double)nblocks * (double)bt.n;
  if (total > (double)max_blocks) { set_error("simt_nmf_loss: partial buffer too small"); return 1; }
  int Rp = (int)round_up(R < 256 ? R : 256, 16);
  size_t smem = (size_t)2 * Rp * kLd * sizeof(float);
  int mode = beta_mode(beta);
  const bool batched = bt.n > 1 || bt.active || bt.scale;
  int rc = with_vtype(V, vdtype, [&](auto Vt) {
    using TV = vtype_t<decltype(Vt)>;
    return with_sel(M, [&](auto Mk) {
      using SEL = sel_t<decltype(Mk)>;
#define NMF_LOSS_B(MD, BATCH, RAGGED)                                                                                       \
  {                                                                                                                         \
    auto kern = simt_loss_kernel<MD, TV, SEL, BATCH, RAGGED>;                                                               \
    NMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                     \
    kern<<<grid, 256, smem, st>>>(Vt, ldv, F, G, Mr, Nc, R, Rp, (float)beta, nchunks, block_partials, Mk, M ? ldm : 0, bt);\
  }
#define NMF_LOSS(MD)                                                                                                        \
  {                                                                                                                         \
    if constexpr (std::is_same<SEL, NoSel>::value) {                                                                        \
      if (bt.rag) { NMF_LOSS_B(MD, true, true); break; }                                                                    \
      if (batched) { NMF_LOSS_B(MD, true, false); break; }                                                                  \
    }                                                                                                                       \
    NMF_LOSS_B(MD, false, false);                                                                                           \
  }
      switch (mode) {
        case kKL: NMF_LOSS(kKL); break;
        case kEU: NMF_LOSS(kEU); break;
        case kIS: NMF_LOSS(kIS); break;
        default: NMF_LOSS(kGeneric); break;
      }
#undef NMF_LOSS
#undef NMF_LOSS_B
      NMF_LAUNCH_CHECK();
      return 0;
    });
  });
  if (rc) return rc;
  return sum_partials(block_partials, nblocks, loss_dev, st, bt.n, bt.active, bt.rag);
}

int simt_nmf_contract_den(const float* F, const float* G, int64_t Mr, int64_t Nc, int R, double beta, int nchunks,
                          float* den, int64_t ldp, int64_t chunk_stride, cudaStream_t st) {
  if (R < 1 || R > 256) { set_error("simt_nmf_contract_den: rank must be in [1, 256]"); return 1; }
  const float bm1 = (float)(beta - 1.0);
  const dim3 grid((unsigned)ceil_div(Mr, kTile), (unsigned)nchunks, 1u);
  const int Rp = 16 * contract_rb(R);
  const size_t smem = (size_t)(2 * Rp + kTile) * kLd * sizeof(float);     // Fs, Gs and the Pp tile
#define NMF_DEN(RBV)                                                                                                 \
  {                                                                                                                  \
    auto kern = simt_contract_kernel<RBV, false, kVFree, float>;                                                     \
    NMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));              \
    kern<<<grid, 256, smem, st>>>(nullptr, 0, F, G, Mr, Nc, R, 0.f, bm1, nchunks, nullptr, den, ldp, chunk_stride,   \
                                  nullptr, 0, Batch{}, nullptr);                                                     \
  } break
  switch (contract_rb(R)) {
    case 1: NMF_DEN(1);
    case 2: NMF_DEN(2);
    case 4: NMF_DEN(4);
    case 8: NMF_DEN(8);
    default: NMF_DEN(16);
  }
#undef NMF_DEN
  NMF_LAUNCH_CHECK();
  return 0;
}

int simt_nmf_contract_num(const void* V, int vdtype, int64_t ldv, int trans, const float* G, int64_t Mr, int64_t Nc, int R,
                          int nchunks, float* num, int64_t chunk_stride, cudaStream_t st, const Batch& bt) {
  if (R < 1 || R > 256) { set_error("simt_nmf_contract_num: rank must be in [1, 256]"); return 1; }
  if (bt.rag) { set_error("simt_nmf_contract_num: a ragged batch is not served"); return 1; }
  unsigned gx;
  if (batch_grid_x(ceil_div(Mr, kTile), bt, "simt_nmf_contract_num", &gx)) return 1;
  const dim3 grid(gx, (unsigned)nchunks, 1u);
  const int Rp = 16 * contract_rb(R);
  const size_t smem = (size_t)(Rp + kTile) * kLd * sizeof(float);           // Gs and the V tile
  const bool batched = bt.n > 1 || bt.active;
  return with_vtype(V, vdtype, [&](auto Vt) {
    using TV = vtype_t<decltype(Vt)>;
#define NMF_NUM_B(RBV, TR, BATCH)                                                                                    \
  {                                                                                                                  \
    auto kern = simt_contract_kernel<RBV, TR, kNumOnly, TV, NoSel, BATCH>;                                           \
    NMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));              \
    kern<<<grid, 256, smem, st>>>(Vt, ldv, nullptr, G, Mr, Nc, R, 0.f, 0.f, nchunks, num, nullptr, R, chunk_stride,  \
                                  nullptr, 0, bt, nullptr);                                                          \
  }
#define NMF_NUM(RBV, TR)                  \
  {                                       \
    if (batched) NMF_NUM_B(RBV, TR, true) \
    else NMF_NUM_B(RBV, TR, false)        \
  }
#define NMF_NUM_RB(RBV)          \
  if (trans) NMF_NUM(RBV, true)  \
  else NMF_NUM(RBV, false)       \
  break
    switch (contract_rb(R)) {
      case 1: NMF_NUM_RB(1);
      case 2: NMF_NUM_RB(2);
      case 4: NMF_NUM_RB(4);
      case 8: NMF_NUM_RB(8);
      default: NMF_NUM_RB(16);
    }
#undef NMF_NUM_RB
#undef NMF_NUM
#undef NMF_NUM_B
    NMF_LAUNCH_CHECK();
    return 0;
  });
}

int64_t simt_plca_fill_blocks(int64_t Mr, int nchunks) { return ceil_div(Mr, kTile) * nchunks; }

int simt_plca_fill_contract(const float* V, int64_t ldv, int trans, const float* F, const float* G, int64_t Mr, int64_t Nc,
                            int R, int nchunks, float* num, float* den, int64_t ldp, int64_t chunk_stride, const uint8_t* M,
                            int64_t ldm, double* qobs_part, cudaStream_t st) {
  if (R < 1) { set_error("simt_plca_fill_contract: rank must be positive"); return 1; }
  if (!M) { set_error("simt_plca_fill_contract: needs the mask"); return 1; }
  const dim3 grid((unsigned)ceil_div(Mr, kTile), (unsigned)nchunks, (unsigned)simt_rank_blocks(R));
  const int Rp = 16 * contract_rb(R);
  const size_t smem = (size_t)(2 * Rp + 2 * kTile) * kLd * sizeof(float);      // Fs, Gs, the V / Pn and mask / Pp tiles
#define NMF_FILL(RBV, TR)                                                                                              \
  {                                                                                                                    \
    auto kern = simt_contract_kernel<RBV, TR, kPlcaFill, float, uint8_t>;                                              \
    NMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                \
    kern<<<grid, 256, smem, st>>>(V, ldv, F, G, Mr, Nc, R, 0.f, 0.f, nchunks, num, den, ldp, chunk_stride, M, ldm,     \
                                  Batch{}, qobs_part);                                                                 \
  }
#define NMF_FILL_RB(RBV)                  \
  if (trans) NMF_FILL(RBV, true)          \
  else NMF_FILL(RBV, false)               \
  break
  switch (contract_rb(R)) {
    case 1: NMF_FILL_RB(1);
    case 2: NMF_FILL_RB(2);
    case 4: NMF_FILL_RB(4);
    case 8: NMF_FILL_RB(8);
    default: NMF_FILL_RB(16);
  }
#undef NMF_FILL_RB
#undef NMF_FILL
  NMF_LAUNCH_CHECK();
  return 0;
}

int simt_nmf_pow_sum(const float* F, const float* G, int64_t Mr, int64_t Nc, int R, double beta, double* block_partials,
                     int max_blocks, int* nblocks, cudaStream_t st) {
  if (R < 1) { set_error("simt_nmf_pow_sum: rank must be positive"); return 1; }
  const int nchunks = loss_chunks(Mr, Nc);
  const dim3 grid((unsigned)ceil_div(Mr, kTile), (unsigned)nchunks);
  *nblocks = (int)(grid.x * grid.y);
  if (*nblocks > max_blocks) { set_error("simt_nmf_pow_sum: partial buffer too small"); return 1; }
  const int Rp = (int)round_up(R < 256 ? R : 256, 16);
  const size_t smem = (size_t)2 * Rp * kLd * sizeof(float);
  auto kern = simt_loss_kernel<kVFree, float>;
  NMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, 256, smem, st>>>(nullptr, 0, F, G, Mr, Nc, R, Rp, (float)beta, nchunks, block_partials, nullptr, 0, Batch{});
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace nmfb200
