// NMFD (1-D convolutive NMF, nmf.py:776-779) on Hopper tensor cores (wgmma) for beta = 1: the three contractions of an update as
// im2col-free SLIDING GEMMs.
//
//   recon : S[c, l]     = sum_{r,t} W[c,r,t] H[r, l-t]           then the ratio epilogue  P~ = (V / (S + eps) - kappa) 2^p  (fp16)
//   wgrad : gW[c, r, t] = sum_l  P~[c, l] H[r, l-t]              (W update: numerator = gW / 2^.. + kappa colsum(H))
//   dgrad : gH[r, j]    = sum_{c,t} W[c,r,t] P~[c, j+t]          (H update: numerator = gH / 2^.. + kappa colsum(W))
//
// Each is a GEMM whose one operand is a plain matrix (TMA, SWIZZLE_128B) and whose other operand is a Toeplitz / Hankel
// matrix: row i of a 128 x 64 tile is the 64-element window of ONE fp16 vector (a padded row of H, or a row of P~) that
// starts one element further than row i - 1 (recon, dgrad) or one element earlier (wgrad).  Nothing of that matrix ever
// exists in global memory: per k-block the TMA warp bulk-copies the ~200-element source window into shared memory and
// the eight producer warps write the 128 x 64 tile from it in the SWIZZLE_128B K-major layout (4-byte shared loads,
// one byte-permute per word for odd shifts, 16-byte stores), 2 threads per row.  The same eight warps then issue wgmma SS
// on it exactly as on a TMA-written tile, 64 rows per warpgroup, with the accumulators in registers; after the k loop they
// are staged through shared memory as fp32 rows for the epilogue warps.
//
// Precision design = the NMF kernel's: fp16 operands with power-of-two scales, fp32 accumulation, the
// ratio tile centred on kappa = sum(V) / sum(WH) so that the K = 8192 ... 131200-term numerator sums are signed and small
// (tensor-core accumulation truncates), kappa * colsum added back in fp32 by the ratio stage (apply_update).
#include "tc_nmfd.cuh"

#include <cuda.h>
#include <cudaTypedefs.h>

#include <algorithm>
#include <cstdlib>
#include <string>

#include "sm90_ptx.cuh"

namespace nmfb200 {

namespace {

constexpr int kM = 128;            // tile rows (two wgmma warpgroups of 64)
constexpr int kKB = 64;            // k-block: 64 fp16 = one 128-byte swizzle row
constexpr int kStages = 3;
constexpr int kWinHalfs = 256;     // source window per k-block: 128 rows + 64 columns + alignment slack (512 bytes)
constexpr int kThreads = 384;      // warp 0 TMA | warps 1-3 idle | warps 4-11 producers + MMA (8-11 also epilogue)

enum : int { kRecon = 0, kReconLoss = 1, kWgrad = 2, kDgrad = 3 };

struct NmfdTcParams {
  int B, C, L, R, T, Lin, Tp;     // Tp = T rounded up to 64
  int Lp;                         // padded row length of Hp16 (halfs); H[b,r,j] sits at column padl + j
  int padl;
  int Lq;                         // row pitch of P16 (halfs), >= L + 72, zero beyond L
  const __half* Hp16;             // [B*R][Lp]
  const __half* P16;              // [B*C][Lq]      (wgrad / dgrad source)
  __half* P16out;                 // recon output
  const float* V;                 // [B][C][L] fp32
  const int* exps;                // {eW, eH, eP}: power-of-two exponents of W16, Hp16, P16
  const float* kappa;             // device scalar
  float* out;                     // wgrad: [nsplit][C][R][T]   dgrad: [nsplit][B][R][Lin]
  double* loss_part;              // recon loss: one partial per CTA
  int nsplit, kb_per_split;
  int r_off;                      // dgrad: first component of this launch (components [r_off, r_off + 128))
};

struct Smem {
  static constexpr int kTile = kM * kKB * 2;                 // 16 KB
  static constexpr int kPlain = 0;
  static constexpr int kToep = kStages * kTile;
  static constexpr int kWin = 2 * kStages * kTile;
  static constexpr int kBar = kWin + kStages * kWinHalfs * 2;
  static constexpr int kNumBars = 4 * kStages + 1;           // win_full, tile_full, empty, win_read per stage + acc_full
  static constexpr int kTmemPtr = kBar + 8 * kNumBars;
  static constexpr int kRed = kTmemPtr + 16;
  static constexpr int kTotal = kRed + 8 * 16;
  // after the k loop the accumulators are staged through [0, kWin) as fp32 rows of up to 128 columns
  static constexpr int kAccPitch = 132;
  static_assert(kM * kAccPitch * 4 <= kWin, "accumulator staging");
};

__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
               : "memory");
}

// One kernel, four roles of the same pipeline (KIND):
//   recon / recon-loss : grid (L tiles, C tiles, B);  plain = A = Wr16 tile (rows c), Toeplitz = B (rows l), N = 128
//   wgrad              : grid (C tiles, R x shift blocks, nsplit);  plain = A = P16 tile (rows c),  Toeplitz = B (rows t of
//                        one block of 128 shifts), N = 128
//   dgrad              : grid (Lin tiles, nsplit, B); Toeplitz = A (rows j), plain = B = Wf16 rows (c R + r_off + n), N = 128;
//                        ranks above 128 take one launch per 128 components
template <int KIND>
__global__ void __launch_bounds__(kThreads, 1)
tcnmfd_kernel(const __grid_constant__ CUtensorMap tmPlain, const NmfdTcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t raw32 = ptx::smem_u32(smem_raw);
  const uint32_t sbase = (raw32 + 1023u) & ~1023u;
  uint8_t* smem_al = smem_raw + (sbase - raw32);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  auto BAR = [&](int i) { return sbase + Smem::kBar + 8u * i; };
  constexpr int B_WIN = 0, B_TILE = kStages, B_EMPTY = 2 * kStages, B_WREAD = 3 * kStages;
  constexpr bool RECON = KIND == kRecon || KIND == kReconLoss;
  const int Rb = min((p.R + 15) & ~15, 128);     // dgrad: B-tile rows loaded per k-block

  if (warp == 0 && lane == 0) {
    ptx::prefetch_tmap(&tmPlain);
    for (int i = 0; i < kStages; ++i) {
      ptx::mbar_init(BAR(B_WIN + i), 1);
      ptx::mbar_init(BAR(B_TILE + i), 8);        // one arrival per producer warp
      ptx::mbar_init(BAR(B_EMPTY + i), 8);       // the MMAs of both warpgroups have completed
      ptx::mbar_init(BAR(B_WREAD + i), 8);       // the 8 producer warps have read the source window of this stage
    }
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
  }
  __syncthreads();

  // ---- what this CTA computes, as a list of k-blocks: (plain-tile coordinates, source vector, window start) -------------
  int nkb, kb0 = 0;
  if (RECON) nkb = p.R * (p.Tp / kKB);
  else { kb0 = (KIND == kWgrad ? blockIdx.z : blockIdx.y) * p.kb_per_split; nkb = p.kb_per_split; }
  const int lkb = (p.L + kKB - 1) / kKB;                    // wgrad: k-blocks per batch element
  const int tkb = p.Tp / kKB;
  const int ntb = (p.T + kM - 1) / kM;                      // wgrad: blocks of 128 shifts (blockIdx.y = r ntb + tb)
  if (KIND == kWgrad) nkb = max(0, min(nkb, p.B * lkb - kb0));
  if (KIND == kDgrad) nkb = max(0, min(nkb, p.C * tkb - kb0));
  // per k-block: returns the plain tile's TMA coordinates (x = column, y = row), the source row pointer and the index of the
  // source element that row 0 / column 0 of the Toeplitz tile reads; `dir` is the step of that index from row to row
  auto kblock = [&](int kb, int& px, int& py, const __half*& src, int& e0) {
    if (RECON) {
      const int r = kb / tkb, kk = kb - r * tkb;            // k = reversed shift t' in [64 kk, 64 kk + 64)
      px = r * p.Tp + kk * kKB; py = blockIdx.y * kM;
      src = p.Hp16 + ((int64_t)blockIdx.z * p.R + r) * p.Lp;
      e0 = p.padl + blockIdx.x * kM - p.Tp + 1 + kk * kKB;  // H index l - t = l - (Tp - 1 - t')
    } else if (KIND == kWgrad) {
      const int g = kb0 + kb, b = g / lkb, lk = g - b * lkb;
      px = lk * kKB; py = b * p.C + blockIdx.x * kM;
      src = p.Hp16 + ((int64_t)b * p.R + blockIdx.y / ntb) * p.Lp;
      e0 = p.padl + lk * kKB - (blockIdx.y % ntb) * kM;     // row i reads H[l - t] of shift t = 128 tb + i: e0 - i
    } else {
      const int g = kb0 + kb, c = g / tkb, kk = g - c * tkb;
      px = kk * kKB; py = c * p.R + p.r_off;
      src = p.P16 + ((int64_t)blockIdx.z * p.C + c) * p.Lq;
      e0 = blockIdx.x * kM + kk * kKB;                      // row j reads P[j + t]
    }
  };
  constexpr int dir = KIND == kWgrad ? -1 : 1;
  // window = source elements [wbeg, wbeg + kWinHalfs), wbeg 8-aligned and <= the smallest index any row reads
  auto win_begin = [&](int e0) { return (dir > 0 ? e0 : e0 - (kM - 1)) & ~7; };

  if (warp == 0) {
    // =========================== TMA: plain operand tile + source window per k-block ==============================
    if (lane == 0) {
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % kStages, ph = (kb / kStages) & 1;
        ptx::mbar_wait(BAR(B_EMPTY + s), ph ^ 1);      // the MMAs that read this stage's tiles have completed ...
        ptx::mbar_wait(BAR(B_WREAD + s), ph ^ 1);      // ... and every producer warp has read its source window
        int px, py, e0; const __half* src;
        kblock(kb, px, py, src, e0);
        const uint32_t plain_bytes = KIND == kDgrad ? (uint32_t)Rb * kKB * 2 : (uint32_t)Smem::kTile;
        ptx::mbar_expect_tx(BAR(B_WIN + s), plain_bytes + kWinHalfs * 2);
        ptx::tma_load_2d(&tmPlain, BAR(B_WIN + s), sbase + Smem::kPlain + s * Smem::kTile, px, py);
        bulk_copy_g2s(sbase + Smem::kWin + s * kWinHalfs * 2, src + win_begin(e0), kWinHalfs * 2, BAR(B_WIN + s));
      }
    }
  } else if (warp >= 4) {
    // =========================== Toeplitz producers: 8 warps, 2 threads per tile row ==================================
    // Then each of the two warpgroups multiplies its 64 rows of the stage: acc[64 x 128] += A[rows] B^T (wgmma SS, the
    // plain tile by TMA and the Toeplitz tile in the same SWIZZLE_128B K-major layout).  dgrad: N = 128 B-rows of which
    // the first Rb were loaded; the columns beyond R are never stored.
    const int pt = threadIdx.x - 128;              // 0..255
    const int row = pt >> 1, half = pt & 1;        // this thread writes columns [32 half, 32 half + 32) of its row
    const int mw = pt >> 7;                        // wgmma warpgroup: tile rows [64 mw, 64 mw + 64)
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < nkb; ++kb) {
      const int s = kb % kStages, ph = (kb / kStages) & 1;
      int px, py, e0; const __half* src;
      kblock(kb, px, py, src, e0);
      const int off = e0 + dir * row - win_begin(e0) + 32 * half;        // first window element this thread reads (>= 0)
      ptx::mbar_wait(BAR(B_WIN + s), ph);                               // window (and plain tile) landed
      const uint32_t win = sbase + Smem::kWin + s * kWinHalfs * 2 + (uint32_t)(off >> 1) * 4;
      uint32_t w[17];
#pragma unroll
      for (int i = 0; i < 17; ++i) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w[i]) : "r"(win + 4 * i));
      const uint32_t sel = (off & 1) ? 0x5432u : 0x3210u;                // odd start: take the upper half of w[i] and the lower of w[i+1]
      uint32_t o[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) o[i] = __byte_perm(w[i], w[i + 1], sel);
      const uint32_t dst = sbase + Smem::kToep + s * Smem::kTile + row * 128;
#pragma unroll
      for (int c16 = 0; c16 < 4; ++c16) {
        const uint32_t chunk = (uint32_t)(4 * half + c16) ^ (uint32_t)(row & 7);      // SWIZZLE_128B
        asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};"
                     ::"r"(dst + (chunk << 4)), "r"(o[4 * c16]), "r"(o[4 * c16 + 1]), "r"(o[4 * c16 + 2]), "r"(o[4 * c16 + 3])
                     : "memory");
      }
      ptx::fence_proxy_async();                    // generic-proxy stores -> visible to the tensor core (async proxy)
      __syncwarp();
      if (lane == 0) { ptx::mbar_arrive(BAR(B_TILE + s)); ptx::mbar_arrive(BAR(B_WREAD + s)); }
      ptx::mbar_wait(BAR(B_TILE + s), ph);                              // every row of the Toeplitz tile written
      const uint32_t plain = sbase + Smem::kPlain + s * Smem::kTile, toep = sbase + Smem::kToep + s * Smem::kTile;
      const uint32_t aBase = (KIND == kDgrad ? toep : plain) + mw * (64 * 128), bBase = KIND == kDgrad ? plain : toep;
      ptx::wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < kKB / 16; ++ks)
        ptx::wgmma_ss_m64n128(acc, ptx::gmma_desc_sw128(aBase + ks * 32, 16, 1024), ptx::gmma_desc_sw128(bBase + ks * 32, 16, 1024), 1u);
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(BAR(B_EMPTY + s));
    }
    // stage the accumulators as fp32 rows (the k loop's tiles are no longer read by anyone once both warpgroups are here)
    float* stg = reinterpret_cast<float*>(smem_al);
    asm volatile("bar.sync 2, 256;" ::: "memory");
    {
      const int r0 = mw * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
      for (int jn = 0; jn < 16; ++jn)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          *reinterpret_cast<float2*>(stg + (r0 + 8 * h) * Smem::kAccPitch + 8 * jn + c0) =
              make_float2(acc[4 * jn + 2 * h], acc[4 * jn + 2 * h + 1]);
    }
    asm volatile("bar.sync 2, 256;" ::: "memory");
    if (warp >= 8) {
      // =========================== epilogue (warps 8-11: one tile row per thread) =====================================
      const int q = warp & 3, r128 = q * 32 + lane;
      const float* arow = stg + r128 * Smem::kAccPitch;
      auto ld16 = [&](int j, uint32_t (&sr)[16]) {
#pragma unroll
        for (int i = 0; i < 16; ++i) sr[i] = __float_as_uint(arow[j * 16 + i]);
      };
      const float sc = exp2f(-(float)(p.exps[KIND == kDgrad ? 0 : (RECON ? 0 : 2)] + p.exps[RECON ? 1 : (KIND == kWgrad ? 1 : 2)]));
      if (RECON) {
        const int c = blockIdx.y * kM + r128, b = blockIdx.z, l0 = blockIdx.x * kM;
        const bool row_ok = c < p.C;
        const float kap = *p.kappa, pscale = exp2f((float)p.exps[2]);
        const float* vrow = p.V + ((int64_t)b * p.C + (row_ok ? c : 0)) * p.L;
        __half* prow = p.P16out + ((int64_t)b * p.C + (row_ok ? c : 0)) * p.Lq;
        double acc = 0.0;
#pragma unroll 1
        for (int j = 0; j < kM / 16; ++j) {
          uint32_t sr[16];
          ld16(j, sr);
          const int l = l0 + j * 16;
          float v[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) v[i] = (row_ok && l + i < p.L) ? vrow[l + i] : 0.f;
          if (KIND == kReconLoss) {
            float a = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const float x = __uint_as_float(sr[i]) * sc;
              if (row_ok && l + i < p.L) a += v[i] * (logf(v[i] + kEps) - logf(x + kEps)) - v[i] + x;     // metrics.py:22
            }
            acc += (double)a;
          } else {
            uint32_t pk[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float x0 = fmaf(__uint_as_float(sr[2 * i]), sc, kEps), x1 = fmaf(__uint_as_float(sr[2 * i + 1]), sc, kEps);
              const float p0 = (v[2 * i] / x0 - kap) * pscale, p1 = (v[2 * i + 1] / x1 - kap) * pscale;      // nmf.py:65, centred
              pk[i] = ptx::pack_f16x2_sat((l + 2 * i < p.L) ? p0 : 0.f, (l + 2 * i + 1 < p.L) ? p1 : 0.f);
            }
            if (row_ok && l < p.Lq) {
              *reinterpret_cast<uint4*>(prow + l) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
              *reinterpret_cast<uint4*>(prow + l + 8) = make_uint4(pk[4], pk[5], pk[6], pk[7]);
            }
          }
        }
        if (KIND == kReconLoss) {
          double* red = reinterpret_cast<double*>(smem_al + Smem::kRed);
          for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
          if (lane == 0) red[q] = acc;
          asm volatile("bar.sync 1, 128;");
          if (q == 0 && lane == 0)
            p.loss_part[((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = (red[0] + red[1]) + (red[2] + red[3]);
        }
      } else if (KIND == kWgrad) {
        const int c = blockIdx.x * kM + r128, r = blockIdx.y / ntb, t0 = (blockIdx.y % ntb) * kM;
        float* dst = p.out + (((int64_t)blockIdx.z * p.C + (c < p.C ? c : 0)) * p.R + r) * p.T + t0;  // [split][C][R][T]
        const bool vec = (p.T & 3) == 0;
#pragma unroll 1
        for (int j = 0; j < kM / 16; ++j) {
          uint32_t sr[16];
          ld16(j, sr);
          if (c < p.C && t0 + j * 16 < p.T) {
            if (vec && t0 + j * 16 + 16 <= p.T) {
#pragma unroll
              for (int i = 0; i < 16; i += 4)
                *reinterpret_cast<float4*>(dst + j * 16 + i) = make_float4(__uint_as_float(sr[i]) * sc, __uint_as_float(sr[i + 1]) * sc,
                                                                           __uint_as_float(sr[i + 2]) * sc, __uint_as_float(sr[i + 3]) * sc);
            } else {
#pragma unroll
              for (int i = 0; i < 16; ++i)
                if (t0 + j * 16 + i < p.T) dst[j * 16 + i] = __uint_as_float(sr[i]) * sc;
            }
          }
        }
      } else {
        const int j = blockIdx.x * kM + r128, b = blockIdx.z;
#pragma unroll 1
        for (int jj = 0; jj < Rb / 16; ++jj) {
          uint32_t sr[16];
          ld16(jj, sr);
          if (j < p.Lin) {
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              const int r = p.r_off + jj * 16 + i;
              if (r < p.R) p.out[(((int64_t)blockIdx.y * p.B + b) * p.R + r) * p.Lin + j] = __uint_as_float(sr[i]) * sc;
            }
          }
        }
      }
    }
  }
}

// ---- operand preparation --------------------------------------------------------------------------------------------------
__device__ __forceinline__ int pow2_exp14(float mx) {
  if (!(mx > 0.f) || !isfinite(mx)) return 0;
  int e;
  frexpf(mx, &e);
  return 14 - e;
}

__global__ void __launch_bounds__(256)
absmax_kernel(const float* __restrict__ x, int64_t n, unsigned int* __restrict__ out) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) m = fmaxf(m, x[i]);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));
}

// colsum[r] = sum over `outer` slabs of `inner` consecutive partials each: part[(o R + r) inner + i]; block r, fixed order.
// The block that finishes LAST also publishes kappa = sum(V) / sum_r colsum_W[r] colsum_H[r] (= sum of the reconstruction,
// nmf.py:776-779) and the exponent of the ratio tile (kappa 2^p in [2^-4, 2^-3)) when no other refresh follows in this call:
// two launches per refresh (prep, fold) instead of three.
struct FoldTail {
  const float* part;        // [(o R + r) inner + i]
  float* colsum;            // [R] of the factor being refreshed
  int outer, R, inner;
  unsigned int* ticket;     // zero between launches
  int do_kappa;
  const double* vsum;
  const float* colsum_all;  // [2 R]: W then H
  float* kappa;
  int* exps;
};

__global__ void __launch_bounds__(256)
fold_colsum_kernel(const FoldTail f) {
  __shared__ float sh[256];
  __shared__ bool is_last;
  const int r = blockIdx.x;
  const int64_t n = (int64_t)f.outer * f.inner;
  float a = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += 256) {
    const int64_t o = i / f.inner, k = i - o * f.inner;
    a += f.part[(o * f.R + r) * f.inner + k];
  }
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    f.colsum[r] = sh[0];
    __threadfence();                                            // this component's sum is visible before the ticket is
    is_last = atomicAdd(f.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last || threadIdx.x != 0) return;
  __threadfence();
  *f.ticket = 0u;
  if (f.do_kappa) {
    double dot = 0.0;
    for (int q = 0; q < f.R; ++q) dot += (double)__ldcg(f.colsum_all + q) * (double)__ldcg(f.colsum_all + f.R + q);
    const float k = (float)(*f.vsum / dot);
    int e = 0;
    const bool ok = k > 0.f && isfinite(k);
    if (ok) { frexpf(k, &e); e = -3 - e; }
    *f.kappa = ok ? k : 0.f;
    f.exps[2] = e;
  }
}

// One pass over W (C, R, T), block c: both fp16 operand copies of this row, scaled by 2^eW (eW from the max of W), written
// 16 bytes per thread and step, plus the row's per-component sums (-> colsum_W, nmf.py:128-131):
//   Wr16[c][r Tp + tt]           = W[c, r, Tp - 1 - tt]        (recon: shifts reversed so that the H window ascends)
//   Wf16[c][r Tp + tt]           = W[c, r, tt]                 (dgrad)
__global__ void __launch_bounds__(256, 8)     // 8 blocks per SM: the 1025 blocks of cfg3 run as one wave
prep_w_kernel(const float* __restrict__ W, int C, int R, int T, int Tp, const unsigned int* __restrict__ absmax,
              int* __restrict__ exps, __half* __restrict__ Wr16, __half* __restrict__ Wf16, float* __restrict__ cs_part) {
  const int e = pow2_exp14(__uint_as_float(*absmax));
  if (blockIdx.x == 0 && threadIdx.x == 0) exps[0] = e;
  const float sc = exp2f((float)e);
  const int c = blockIdx.x;
  const float* Wg = W + (int64_t)c * R * T;
  auto w_at = [&](int r, int t) { return (r < R && t >= 0 && t < T) ? Wg[r * T + t] * sc : 0.f; };
  auto pack8 = [&](const float (&v)[8]) {
    __half2 h[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    return *reinterpret_cast<const uint4*>(h);
  };
  const int64_t rowlen = (int64_t)R * Tp;
  for (int i8 = threadIdx.x; i8 < R * Tp / 8; i8 += 256) {
    const int i = i8 * 8, r = i / Tp, tt = i - r * Tp;
    float f[8], rv[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { f[k] = w_at(r, tt + k); rv[k] = w_at(r, Tp - 1 - tt - k); }
    *reinterpret_cast<uint4*>(Wf16 + c * rowlen + i) = pack8(f);
    *reinterpret_cast<uint4*>(Wr16 + c * rowlen + i) = pack8(rv);
  }
  // per-component sums of this row: warp w takes r = w, w + 8, ...; fixed order
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < R; r += 8) {
    float a = 0.f;
    for (int t = lane; t < T; t += 32) a += Wg[r * T + t];
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) cs_part[(int64_t)c * R + r] = a;
  }
}

// H (B, R, Lin) fp32 -> Hp16 (B R rows x Lp): H[b,r,j] 2^eH at column padl + j (margins stay zero), 2048 elements per
// block, + the block's partial sum (-> colsum_H, nmf.py:122-125).  grid (chunks, B R)
__global__ void __launch_bounds__(256)
prep_h_kernel(const float* __restrict__ H, int Lin, int Lp, int padl, const unsigned int* __restrict__ absmax,
              int* __restrict__ exps, __half* __restrict__ Hp16, float* __restrict__ cs_part) {
  __shared__ float sh[8];
  const int e = pow2_exp14(__uint_as_float(*absmax));
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) exps[1] = e;
  const float sc = exp2f((float)e);
  const int64_t row = blockIdx.y;
  const int j = blockIdx.x * 2048 + threadIdx.x * 8;
  float a = 0.f;
  if (j < Lin) {
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { v[k] = j + k < Lin ? H[row * Lin + j + k] : 0.f; a += v[k]; v[k] *= sc; }
    __half2 h[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
    *reinterpret_cast<uint4*>(Hp16 + row * Lp + padl + j) = *reinterpret_cast<const uint4*>(h);
  }
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += sh[i];
    cs_part[row * gridDim.x + blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(256)
vsum_kernel(const float* __restrict__ V, int64_t n, double* __restrict__ part) {
  __shared__ double sh[8];
  double a = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) a += (double)V[i];
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0.0; for (int i = 0; i < 8; ++i) t += sh[i]; part[blockIdx.x] = t; }
}

PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
  return fn;
}

int make_tmap2(CUtensorMap* m, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  auto fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return 2; }
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (nmfd) failed with code " + std::to_string((int)r)); return 2; }
  return 0;
}

}  // namespace

struct TcNmfdState {
  NmfdShape d{};
  int Tp = 0, Lp = 0, padl = 0, Lq = 0, Cpad = 0;
  __half *Wr16 = nullptr, *Wf16 = nullptr, *Hp16 = nullptr, *P16 = nullptr;
  float* part = nullptr;            // wgrad / dgrad split partials
  int64_t part_floats = 0;
  unsigned int* absmax = nullptr;   // [2]: max of W, max of H (float bits; written by absmax_kernel or by the ratio stage)
  float* colsum = nullptr;          // [2][R]: colsum_W | colsum_H
  float* cs_part = nullptr;         // per-row / per-block partial sums of the factor being refreshed
  bool w_fresh = false, h_fresh = false;      // the fp16 copies / column sums of W, H match the fp32 factor
  bool aw_valid = false, ah_valid = false;    // absmax[0], absmax[1] hold the max of the current W, H
  int* exps = nullptr;              // {eW, eH, eP}
  float* kappa = nullptr;
  double* vsum = nullptr;           // [1] + [256] partials
  double* loss_part = nullptr;
  int loss_blocks = 0;
  int ws_w = 1, ws_h = 1;           // split counts of wgrad / dgrad
  int kbs_w = 0, kbs_h = 0;
  CUtensorMap tmWr, tmWf, tmP;
  bool attr_set = false;
};

bool tc_nmfd_supported(const NmfdShape& d, double beta) {
  // wgrad's grid.y = R x blocks of 128 shifts
  return beta == 1.0 && d.R >= 1 && d.R <= 256 && d.T >= 1 && d.L >= d.T && (int64_t)d.R * ceil_div(d.T, kM) <= 65535;
}

void tc_nmfd_destroy(TcNmfdState* s) {
  if (!s) return;
  cudaFree(s->Wr16); cudaFree(s->Wf16); cudaFree(s->Hp16); cudaFree(s->P16); cudaFree(s->part); cudaFree(s->absmax); cudaFree(s->colsum); cudaFree(s->cs_part);
  cudaFree(s->exps); cudaFree(s->kappa); cudaFree(s->vsum); cudaFree(s->loss_part);
  delete s;
}

int tc_nmfd_create(TcNmfdState** out, const NmfdShape& d) {
  *out = nullptr;
  TcNmfdState* s = new TcNmfdState();
  s->d = d;
  s->Tp = (int)round_up(d.T, kKB);
  s->padl = (int)round_up(s->Tp + 136, 8);                       // every window start >= 0
  s->Lp = (int)round_up((int64_t)s->padl + round_up((int64_t)d.L, 2048) + 256 + kWinHalfs + 136, 8);
  s->Lq = (int)round_up(round_up((int64_t)d.L, 2048) + 1024 + s->Tp + kKB + kWinHalfs + 8, 8);
  s->Cpad = (int)round_up(d.C, kM);
  const int lkb = (int)ceil_div(d.L, kKB), tkb = s->Tp / kKB;
  // split the K loops of wgrad / dgrad so that the grid is a few waves of 132 CTAs
  const int64_t tiles_w = ceil_div(d.C, kM) * d.R * ceil_div(d.T, kM), tiles_h = ceil_div(d.Lin, kM) * d.B;
  int64_t kb_w = (int64_t)d.B * lkb, kb_h = (int64_t)d.C * tkb;
  s->ws_w = (int)std::max<int64_t>(1, std::min<int64_t>(kb_w / 8, ceil_div(132 * 4, tiles_w)));
  s->ws_h = (int)std::max<int64_t>(1, std::min<int64_t>(kb_h / 8, ceil_div(132 * 4, tiles_h)));
  s->kbs_w = (int)ceil_div(kb_w, s->ws_w); s->ws_w = (int)ceil_div(kb_w, s->kbs_w);
  s->kbs_h = (int)ceil_div(kb_h, s->ws_h); s->ws_h = (int)ceil_div(kb_h, s->kbs_h);
  const int hs = s->ws_h;
  const int64_t pw = (int64_t)s->ws_w * d.C * d.R * d.T, ph = (int64_t)hs * d.B * d.R * d.Lin;
  s->part_floats = pw > ph ? pw : ph;
  s->loss_blocks = (int)(ceil_div(d.L, kM) * ceil_div(d.C, kM) * d.B);
  const size_t wbytes = (size_t)s->Cpad * d.R * s->Tp * 2, hbytes = (size_t)d.B * d.R * s->Lp * 2;
  const size_t pbytes = ((size_t)d.B * d.C + 1) * s->Lq * 2;
  cudaError_t e = cudaSuccess;
  if (e == cudaSuccess) e = cudaMalloc(&s->Wr16, wbytes);
  if (e == cudaSuccess) e = cudaMalloc(&s->Wf16, wbytes);
  if (e == cudaSuccess) e = cudaMalloc(&s->Hp16, hbytes);
  if (e == cudaSuccess) e = cudaMalloc(&s->P16, pbytes);
  if (e == cudaSuccess) e = cudaMalloc(&s->part, (size_t)s->part_floats * 4);
  if (e == cudaSuccess) e = cudaMalloc(&s->absmax, 2 * sizeof(unsigned int));
  if (e == cudaSuccess) e = cudaMalloc(&s->colsum, 2 * (size_t)d.R * sizeof(float));
  {
    const int64_t np = std::max<int64_t>((int64_t)d.C * d.R, (int64_t)d.B * d.R * ceil_div(d.Lin, 2048));
    if (e == cudaSuccess) e = cudaMalloc(&s->cs_part, (size_t)np * sizeof(float));
  }
  if (e == cudaSuccess) e = cudaMalloc(&s->exps, 8 * sizeof(int));          // [0..3] exponents, [4..5] fold tickets
  if (e == cudaSuccess) e = cudaMemset(s->exps, 0, 8 * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&s->kappa, sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&s->vsum, 257 * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&s->loss_part, (size_t)s->loss_blocks * sizeof(double));
  if (e == cudaSuccess) e = cudaMemset(s->Wr16, 0, wbytes);
  if (e == cudaSuccess) e = cudaMemset(s->Wf16, 0, wbytes);
  if (e == cudaSuccess) e = cudaMemset(s->Hp16, 0, hbytes);
  if (e == cudaSuccess) e = cudaMemset(s->P16, 0, pbytes);
  if (e == cudaSuccess) e = cudaMemset(s->exps, 0, 4 * sizeof(int));
  if (e != cudaSuccess) {
    tc_nmfd_destroy(s);
    set_error(std::string("tc_nmfd_create: ") + cudaGetErrorString(e));
    return 2;
  }
  int rc = 0;
  rc |= make_tmap2(&s->tmWr, s->Wr16, s->Cpad, (int64_t)d.R * s->Tp, (int64_t)d.R * s->Tp, kM);
  // dgrad reads Wf16 as (C R) rows of Tp columns, up to 128 rows (components) per tile
  const int Rb = (int)std::min<int64_t>((d.R + 15) & ~15, 128);
  rc |= make_tmap2(&s->tmWf, s->Wf16, (int64_t)s->Cpad * d.R, s->Tp, s->Tp, Rb);
  rc |= make_tmap2(&s->tmP, s->P16, (int64_t)d.B * d.C, s->Lq, s->Lq, kM);
  if (rc) { tc_nmfd_destroy(s); return 2; }
  *out = s;
  return 0;
}

int tc_nmfd_set_target(TcNmfdState* s, const float* V, double* vsum_host, cudaStream_t st) {
  const int64_t n = (int64_t)s->d.B * s->d.C * s->d.L;
  vsum_kernel<<<256, 256, 0, st>>>(V, n, s->vsum + 1);
  NMF_LAUNCH_CHECK();
  int rc = sum_partials(s->vsum + 1, 256, s->vsum, st);
  if (rc) return rc;
  NMF_CUDA_CHECK(cudaMemcpyAsync(vsum_host, s->vsum, sizeof(double), cudaMemcpyDeviceToHost, st));
  NMF_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

namespace {

template <int KIND>
int launch(TcNmfdState* s, const CUtensorMap& tm, dim3 grid, NmfdTcParams& p, cudaStream_t st) {
  auto kern = tcnmfd_kernel<KIND>;
  static bool attr = false;
  const int smem = Smem::kTotal + 1024;
  if (!attr) {
    NMF_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr = true;
  }
  kern<<<grid, kThreads, smem, st>>>(tm, p);
  NMF_LAUNCH_CHECK();
  return 0;
}

NmfdTcParams base_params(TcNmfdState* s, const float* V) {
  NmfdTcParams p{};
  p.B = s->d.B; p.C = s->d.C; p.L = s->d.L; p.R = s->d.R; p.T = s->d.T; p.Lin = s->d.Lin; p.Tp = s->Tp;
  p.Lp = s->Lp; p.padl = s->padl; p.Lq = s->Lq;
  p.Hp16 = s->Hp16; p.P16 = s->P16; p.P16out = s->P16; p.V = V; p.exps = s->exps; p.kappa = s->kappa;
  p.out = s->part; p.loss_part = s->loss_part; p.nsplit = 1; p.kb_per_split = 0;
  return p;
}

// arguments of the fold launch after a preparation launch: fold `outer x R x inner` partial sums into colsum[which], then kappa if this is the
// last refresh of the call
FoldTail fold_tail_args(TcNmfdState* s, int which, int outer, int inner, int do_kappa) {
  FoldTail f{};
  f.part = s->cs_part; f.colsum = s->colsum + (which ? s->d.R : 0); f.outer = outer; f.R = s->d.R; f.inner = inner;
  f.ticket = reinterpret_cast<unsigned int*>(s->exps + 4 + which); f.do_kappa = do_kappa;
  f.vsum = s->vsum; f.colsum_all = s->colsum; f.kappa = s->kappa; f.exps = s->exps;
  return f;
}

// bring the fp16 operand copies, column sums (and with them kappa) up to date with the fp32 factors: only what changed
int refresh(TcNmfdState* s, const float* W, const float* H, cudaStream_t st) {
  const NmfdShape& d = s->d;
  if (!s->w_fresh) {
    if (!s->aw_valid) {
      NMF_CUDA_CHECK(cudaMemsetAsync(s->absmax, 0, sizeof(unsigned int), st));
      absmax_kernel<<<256, 256, 0, st>>>(W, (int64_t)d.C * d.R * d.T, s->absmax);
      NMF_LAUNCH_CHECK();
      s->aw_valid = true;
    }
    prep_w_kernel<<<d.C, 256, 0, st>>>(W, d.C, d.R, d.T, s->Tp, s->absmax, s->exps, s->Wr16, s->Wf16, s->cs_part);
    NMF_LAUNCH_CHECK();
    fold_colsum_kernel<<<d.R, 256, 0, st>>>(fold_tail_args(s, 0, d.C, 1, /*do_kappa=*/s->h_fresh));
    NMF_LAUNCH_CHECK();
    s->w_fresh = true;
  }
  if (!s->h_fresh) {
    if (!s->ah_valid) {
      NMF_CUDA_CHECK(cudaMemsetAsync(s->absmax + 1, 0, sizeof(unsigned int), st));
      absmax_kernel<<<256, 256, 0, st>>>(H, (int64_t)d.B * d.R * d.Lin, s->absmax + 1);
      NMF_LAUNCH_CHECK();
      s->ah_valid = true;
    }
    const int nch = (int)ceil_div(d.Lin, 2048);
    dim3 gh((unsigned)nch, (unsigned)(d.B * d.R));
    prep_h_kernel<<<gh, 256, 0, st>>>(H, d.Lin, s->Lp, s->padl, s->absmax + 1, s->exps, s->Hp16, s->cs_part);
    NMF_LAUNCH_CHECK();
    fold_colsum_kernel<<<d.R, 256, 0, st>>>(fold_tail_args(s, 1, d.B, nch, /*do_kappa=*/1));
    NMF_LAUNCH_CHECK();
    s->h_fresh = true;
  }
  return 0;
}

}  // namespace

int tc_nmfd_recon(TcNmfdState* s, const float* V, const float* W, const float* H, bool loss, double* loss_dev,
                  cudaStream_t st) {
  int rc = refresh(s, W, H, st);
  if (rc) return rc;
  NmfdTcParams p = base_params(s, V);
  dim3 grid((unsigned)ceil_div(s->d.L, kM), (unsigned)ceil_div(s->d.C, kM), (unsigned)s->d.B);
  if (loss) {
    rc = launch<kReconLoss>(s, s->tmWr, grid, p, st);
    if (rc) return rc;
    return sum_partials(s->loss_part, (int)(grid.x * grid.y * grid.z), loss_dev, st);
  }
  return launch<kRecon>(s, s->tmWr, grid, p, st);
}

// numerator partials of the W update from the P16 written by the last recon: [*nsplit][C][R][T] fp32
int tc_nmfd_wgrad(TcNmfdState* s, const float** part, int* nsplit, cudaStream_t st) {
  NmfdTcParams p = base_params(s, nullptr);
  p.nsplit = s->ws_w; p.kb_per_split = s->kbs_w;
  // one CTA per (128 rows c, component r, block of 128 shifts t, split): the Toeplitz tile holds 128 shifts
  dim3 grid((unsigned)ceil_div(s->d.C, kM), (unsigned)(s->d.R * ceil_div(s->d.T, kM)), (unsigned)s->ws_w);
  int rc = launch<kWgrad>(s, s->tmP, grid, p, st);
  *part = s->part; *nsplit = s->ws_w;
  return rc;
}

int tc_nmfd_dgrad(TcNmfdState* s, const float** part, int* nsplit, cudaStream_t st) {
  NmfdTcParams p = base_params(s, nullptr);
  p.nsplit = s->ws_h; p.kb_per_split = s->kbs_h;
  dim3 grid((unsigned)ceil_div(s->d.Lin, kM), (unsigned)s->ws_h, (unsigned)s->d.B);
  int rc = 0;
  for (p.r_off = 0; rc == 0 && p.r_off < s->d.R; p.r_off += 128) rc = launch<kDgrad>(s, s->tmWf, grid, p, st);
  *part = s->part; *nsplit = s->ws_h;
  return rc;
}

const float* tc_nmfd_kappa(const TcNmfdState* s) { return s->kappa; }
const float* tc_nmfd_colsum(const TcNmfdState* s) { return s->colsum; }

// The caller is about to overwrite a factor (which = 0: W, 1: H) with its ratio stage: returns the slot the stage should
// atomicMax the new values into (zeroed here), so the next refresh needs no separate pass for the operand exponent.
unsigned int* tc_nmfd_begin_update(TcNmfdState* s, int which, cudaStream_t st) {
  unsigned int* slot = s->absmax + which;
  if (cudaMemsetAsync(slot, 0, sizeof(unsigned int), st) != cudaSuccess) return nullptr;
  if (which == 0) { s->w_fresh = false; s->aw_valid = true; } else { s->h_fresh = false; s->ah_valid = true; }
  return slot;
}

// a factor was changed by someone else: everything derived from it is stale
void tc_nmfd_mark_dirty(TcNmfdState* s) {
  s->w_fresh = s->h_fresh = false;
  s->aw_valid = s->ah_valid = false;
}

// report (and clear) a recorded mbarrier wait abort of the NMFD kernels; the caller has synchronised the stream
int tc_nmfd_check_wait_abort() {
  unsigned int h[8] = {0};
  if (cudaMemcpyFromSymbol(h, ptx::g_wait_abort, sizeof(h)) != cudaSuccess) return -1;
  if (h[0]) {
    fprintf(stderr, "nmf_b200: NMFD mbarrier wait aborted: block %u thread %u bar_addr %u parity %u\n", h[1], h[2], h[3], h[4]);
    unsigned int z[8] = {0};
    cudaMemcpyToSymbol(ptx::g_wait_abort, z, sizeof(z));
    return 1;
  }
  return 0;
}

}  // namespace nmfb200
