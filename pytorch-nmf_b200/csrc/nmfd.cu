// NMFD / NMF2D / NMF3D (convolutive NMF over one to three axes) contractions as im2col-free sliding GEMMs on CUDA cores, fp32.
//
//   recon : WH[b,c,x]   = sum_{r,t} W[c,r,t] H[b,r,x-t]          nmf.py:776-779, :861-865, :938-942 (flipped kernel, full pad)
//   wgrad : gW[c,r,t]   = sum_{b,x} G[b,c,x] H[b,r,x-t]          autograd of the above w.r.t. W
//   dgrad : gH[b,r,j]   = sum_{c,t} W[c,r,t] G[b,c,j+t]          autograd of the above w.r.t. H
//
// x, t, j are multi-indices over the convolved axes.  The LAST axis is the sliding axis of the kernels; the outer axes
// (NmfdShape::X1, X2 / T1, T2) are loops: recon and dgrad loop over the outer kernel offsets, wgrad over the outer positions
// ("lines").  No Toeplitz/im2col matrix is ever formed: each CTA stages contiguous windows of the shifted operand in shared
// memory and every thread slides a 4-element register window across its line (one shared load + one float4 load per 16
// FMAs).
//
// Tile shapes follow the problem.  A thread owns 4 rows x 4 columns of the output tile; the row tile MT (channels for recon
// and wgrad, components for dgrad) is 4 ... 64, and the 256 / (MT / 4) thread columns that remain cover
//   recon / dgrad: 64 positions of the sliding axis on each of 64 / MT consecutive outer lines,
//   wgrad        : the offsets t of several components r -- and, when those do not fill the block, of several outer kernel
//                  offsets (t1, t2) -- at once,
// so a 3-channel target or a 16-tap kernel does not leave most of the block idle.
#include "common.cuh"

namespace nmfb200 {

namespace {

constexpr int kLT = 64;    // positions of the sliding axis per line tile
constexpr int kTK = 32;    // k-chunk (shifts or samples) per stage

template <int MODE>
__device__ __forceinline__ void phi_d(float v, float s, float bm2, float bm1, float& pn, float& pp) {
  if (MODE == kKL) { pn = v / (s + kEps); pp = 0.f; }
  else if (MODE == kEU) { pn = v; pp = s; }
  else if (MODE == kIS) { float r = 1.0f / (s + kEps); pp = r; pn = (r * r) * v; }
  else { float x = s + kEps; pn = powf(x, bm2) * v; pp = powf(x, bm1); }
}

template <int MODE>
__device__ __forceinline__ float loss_term_d(float v, float s, float beta) {
  if (MODE == kKL) return v * (logf(v + kEps) - logf(s + kEps)) - v + s;
  if (MODE == kEU) { float d = s - v; return 0.5f * d * d; }
  if (MODE == kIS) { float te = v + kEps, xe = s + kEps; return te / xe - logf(te) + logf(xe) - 1.0f; }
  float x = s + kEps, t = beta < 0.f ? v + kEps : v, bm = beta - 1.0f;
  return (powf(t, beta) + bm * powf(x, beta) - beta * t * powf(x, bm)) / (beta * bm);
}

__device__ __forceinline__ double block_sum_d(double v, double* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) sh[w] = v;
  __syncthreads();
  double t = 0.0;
  if (w == 0) {
    t = l < 8 ? sh[l] : 0.0;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  }
  return t;
}

template <int MT>
struct Geo {
  static constexpr int TY = MT / 4;          // thread rows (4 output rows each)
  static constexpr int TX = 256 / TY;        // thread columns (4 output columns each)
  static constexpr int XT = TX / 16;         // outer lines per block (recon / dgrad): 16 thread columns = 64 positions a line
  static constexpr int NCOL = 4 * TX;        // output columns per block (wgrad)
  static constexpr int PAD = MT + 4;         // shared pitch of the row-tile operand
  static constexpr int NTO = MT <= 16 ? 8 : 1;               // wgrad: outer kernel offsets a block may cover
  static constexpr int HS = (NCOL / 4) * (4 + kTK);          // wgrad: floats of H windows (worst case: 4 offsets per component)
};

// ---- recon (FWD) and dgrad (!FWD): out[m, pos] = sum_{k, t} A[m, k, t] X[k, pos -/+ t] ---------------------------------------
//   FWD : m = c, k = r, X = H, shift -t, zero outside H; the epilogue applies phi against V (or reduces the loss)
//   !FWD: m = r, k = c in this block's split, X = G, shift +t; the epilogue writes the partial sums of this split
// grid (line tiles * line groups, row tiles * nsplit, batch elements [b0, b0 + gridDim.z)), 256 threads: batches beyond the
// 65535 of grid.z take several launches
// BATCH (NoSel only, nmfb200_nmfnd_batched_create): the grid-z lines are bt.n problems of s.B lines each, problem after
// problem.  A block of problem `prob` reads A + prob bt.f, X + prob bt.g and its target at V + prob bt.v, writes its Pn / Pp
// (FWD) or its dgrad partials at + prob bt.p (the dgrad slab of one split holds every problem's) and its loss partials as
// the contiguous run a single launch of that problem writes; otherwise it runs the single problem's plan and arithmetic.
// RAGGED (BATCH, bt.rag; s the padded shape): problem `prob` runs the plan of its own lengths rag[prob].rows / .lin along
// the sliding axis.  It reads H (FWD) and V in their padded layouts up to those lengths, and the ratio tiles (!FWD) in its
// own compact layout at + rag[prob].pn; it writes its Pn / Pp there, its dgrad partials at + rag[prob].part in the single
// problem's [split][B][R][h_inner] layout and its loss partials at + rag[prob].loss_part.  Its blocks past its own grid x
// (rag[prob].gx) or dgrad splits (rag[prob].nch[1]) exit at once.
struct SlideArgs {
  const float* A;            // W
  const float* X;            // H (FWD) or G
  int M, K;                  // rows of the output, size of the reduced dimension
  int64_t sm, sk;            // strides of A over m and k (elements); the offset (t1, t2, t) is contiguous
  int nsplit;                // !FWD: splits of k
  const void* V; float beta; float* Pn; float* Pp; double* block_partials;      // FWD epilogue (V: TV elements)
  const void* mask;          // FWD, SEL: the observed cells or the weights (SEL elements, V's layout)
  float* out;                // !FWD: [split][B][R][h_inner]
  int b0;                    // first batch element of this launch
};

// SEL (FWD only): a fit on the observed cells -- at a missing cell V is not read, Pn = Pp = 0 and the loss adds nothing;
// Pp is written at every beta (beta 1: the mask as 0 / 1), so wgrad / dgrad of Pp give the denominators.  A weighted fit
// treats the cells of weight 0 as missing and multiplies Pn, Pp and the loss term by the weight elsewhere (beta 1: Pp = w).
// kPlcaFill (FWD, !LOSS, fp32 V, the uint8 mask, one problem; a masked PLCA fit): Pn = V / (WH + eps) and Pp = 0 at an
// observed cell, Pn = 0 and Pp = WH / (WH + eps) at a missing one (V not read), and, when a.block_partials is set, each
// block's sum of WH over its observed cells into the loss partial the LOSS pass of this launch would write.
template <int MT, bool FWD, int MODE, bool LOSS, typename TV, typename SEL = NoSel, bool BATCH = false, bool RAGGED = false>
__global__ void __launch_bounds__(256)
nmfd_slide_kernel(NmfdShape s, SlideArgs a, Batch bt) {
  constexpr bool MASK = !std::is_same<SEL, NoSel>::value;
  constexpr bool WEIGHT = kWeighted<SEL>;
  constexpr bool FILL = (MODE == kPlcaFill);
  static_assert(!FILL || (FWD && !LOSS && std::is_same<SEL, uint8_t>::value && std::is_same<TV, float>::value && !BATCH),
                "kPlcaFill: the FWD pass of one problem, fp32 V, the uint8 mask");
  static_assert(!RAGGED || BATCH, "RAGGED: a batch");
  using G = Geo<MT>;
  const int hpitch = s.Lin, vpitch = s.L;     // the padded pitches of H and V (RAGGED: s then holds the problem's lengths)
  int gx = 0;                                 // RAGGED: the problem's grid x
  if constexpr (RAGGED) {
    const RaggedProblem& rp = bt.rag[(a.b0 + (int)blockIdx.z) / s.B];
    s.L = (int)rp.rows; s.Lin = rp.lin;
    gx = rp.gx[FWD ? 0 : 1];
    if ((int)blockIdx.x >= gx) return;
    if (!FWD) {
      a.nsplit = rp.nch[1];
      if ((int)blockIdx.y >= a.nsplit * ((a.M + MT - 1) / MT)) return;
    }
  }
  constexpr int WIN = kLT + kTK;                          // window pitch per line (kLT + kTK - 1 elements used)
  __shared__ __align__(16) float As[kTK * G::PAD];        // As[tt][m]
  __shared__ float Xs[G::XT * WIN];
  __shared__ double red[8];
  const int tid = threadIdx.x, tx = tid % G::TX, ty = tid / G::TX;
  const int lt = tx & 15, xl = tx >> 4;
  const int OUT = FWD ? s.X1 * s.X2 : s.J1() * s.J2();    // outer lines of the output
  const int O2 = FWD ? s.X2 : s.J2();
  const int LOUT = FWD ? s.L : s.Lin;                     // output length along the sliding axis
  const int nlt = (LOUT + kLT - 1) / kLT;
  const int lg = blockIdx.x / nlt;
  const int l0 = (blockIdx.x - lg * nlt) * kLT;
  const int mtiles = (a.M + MT - 1) / MT;
  const int split = blockIdx.y / mtiles;
  const int m0 = (blockIdx.y - split * mtiles) * MT;
  int b = a.b0 + blockIdx.z;
  float sc = 1.f;                 // BATCH, KL loss: the problem's bt.scale
  if constexpr (BATCH) {          // the single-problem instantiations compile none of this
    const int prob = b / s.B;
    if (batch_skips(bt.active, prob)) return;
    if (LOSS && MODE == kKL && bt.scale) sc = bt.scale[prob];
    b -= prob * s.B;
    if constexpr (RAGGED) {
      const RaggedProblem& rp = bt.rag[prob];
      a.A += prob * bt.f;
      if (FWD) {
        a.X += prob * bt.g;
        a.V = static_cast<const TV*>(a.V) + prob * bt.v;
        a.Pn += rp.pn; a.Pp += rp.pn;
        if (LOSS) a.block_partials += rp.loss_part;
      } else {
        a.X += rp.pn;
        a.out += rp.part;
      }
    } else {
      a.A += prob * bt.f; a.X += prob * bt.g;
      if (FWD) {
        a.V = static_cast<const TV*>(a.V) + prob * bt.v;
        a.Pn += prob * bt.p; a.Pp += prob * bt.p;
        if (LOSS) a.block_partials += (int64_t)prob * s.B * gridDim.y * gridDim.x;
      } else {
        a.out += prob * bt.p;
      }
    }
  }
  const int kps = (a.K + a.nsplit - 1) / a.nsplit;
  const int kbeg = split * kps, kend = min(a.K, kbeg + kps);
  const int J1 = s.J1(), J2 = s.J2();
  const int nouter = s.T1 * s.T2;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int ko = kbeg * nouter; ko < kend * nouter; ++ko) {
    const int k = ko / nouter, to = ko - k * nouter;
    const int t1 = to / s.T2, t2 = to - t1 * s.T2;
    for (int t0 = 0; t0 < s.T; t0 += kTK) {
      __syncthreads();
      for (int idx = tid; idx < MT * kTK; idx += 256) {
        const int m = idx / kTK, tt = idx - m * kTK;
        float w = 0.f;
        if (m0 + m < a.M && t0 + tt < s.T) w = a.A[(int64_t)(m0 + m) * a.sm + (int64_t)k * a.sk + (int64_t)to * s.T + t0 + tt];
        As[tt * G::PAD + m] = w;
      }
      for (int idx = tid; idx < G::XT * (WIN - 1); idx += 256) {
        const int line = idx / (WIN - 1), i = idx - line * (WIN - 1);
        const int o = lg * G::XT + line;
        const int o1 = o / O2, o2 = o - o1 * O2;
        float x = 0.f;
        if (o < OUT) {
          if (FWD) {
            const int j1 = o1 - t1, j2 = o2 - t2, src = l0 - t0 - (kTK - 1) + i;      // window index of (lj, tt): lj - tt + kTK - 1
            if (j1 >= 0 && j1 < J1 && j2 >= 0 && j2 < J2 && src >= 0 && src < s.Lin)
              x = a.X[((((int64_t)b * a.K + k) * J1 + j1) * J2 + j2) * hpitch + src];
          } else {
            const int src = l0 + t0 + i;                                              // window index of (jj, tt): jj + tt
            if (src < s.L) x = a.X[((((int64_t)b * a.K + k) * s.X1 + (o1 + t1)) * s.X2 + (o2 + t2)) * s.L + src];
          }
        }
        Xs[line * WIN + i] = x;
      }
      __syncthreads();
      const float* xs = Xs + xl * WIN + 4 * lt;
      const int tmax = min(kTK, s.T - t0);
      float h[4];
      if (FWD) {
        h[0] = xs[kTK]; h[1] = xs[kTK + 1]; h[2] = xs[kTK + 2];
#pragma unroll 8
        for (int tt = 0; tt < tmax; ++tt) {
          h[3] = h[2]; h[2] = h[1]; h[1] = h[0];
          h[0] = xs[kTK - 1 - tt];
          const float4 av4 = *reinterpret_cast<const float4*>(&As[tt * G::PAD + 4 * ty]);
          const float av[4] = {av4.x, av4.y, av4.z, av4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], h[j], acc[i][j]);
        }
      } else {
        h[1] = xs[0]; h[2] = xs[1]; h[3] = xs[2];
#pragma unroll 8
        for (int tt = 0; tt < tmax; ++tt) {
          h[0] = h[1]; h[1] = h[2]; h[2] = h[3];
          h[3] = xs[3 + tt];
          const float4 av4 = *reinterpret_cast<const float4*>(&As[tt * G::PAD + 4 * ty]);
          const float av[4] = {av4.x, av4.y, av4.z, av4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], h[j], acc[i][j]);
        }
      }
    }
  }

  const int o = lg * G::XT + xl;
  if (FWD) {
    const float bm2 = a.beta - 2.0f, bm1 = a.beta - 1.0f;
    float local = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = m0 + 4 * ty + i;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int l = l0 + 4 * lt + j;
        if (c < s.C && l < s.L && o < OUT) {
          const int64_t off = (((int64_t)b * s.C + c) * OUT + o) * s.L + l;
          const int64_t voff = RAGGED ? (((int64_t)b * s.C + c) * OUT + o) * vpitch + l : off;     // V's padded layout
          if constexpr (WEIGHT) {
            const float w = static_cast<const float*>(a.mask)[off];
            if (w == 0.f) {
              if (!LOSS) { a.Pn[off] = 0.f; a.Pp[off] = 0.f; }
              continue;
            }
            const float v = to_f32(static_cast<const TV*>(a.V)[voff]);
            if (LOSS) {
              local += MODE == kEU ? loss_term_w<kEU>(v, acc[i][j], a.beta, w) : w * loss_term_d<MODE>(v, acc[i][j], a.beta);
            } else {
              float pn, pp;
              phi_d<MODE>(v, acc[i][j], bm2, bm1, pn, pp);
              a.Pn[off] = pn * w;
              a.Pp[off] = MODE != kKL ? pp * w : w;
            }
            continue;
          }
          if (MASK && !static_cast<const uint8_t*>(a.mask)[off]) {
            if (FILL) { a.Pn[off] = 0.f; a.Pp[off] = acc[i][j] / (acc[i][j] + kEps); }
            else if (!LOSS) { a.Pn[off] = 0.f; a.Pp[off] = 0.f; }
            continue;
          }
          const float v = to_f32(static_cast<const TV*>(a.V)[voff]);
          if (FILL) {
            a.Pn[off] = v / (acc[i][j] + kEps);
            a.Pp[off] = 0.f;
            local += acc[i][j];
          } else if (LOSS) {
            if (BATCH && MODE == kKL) local += loss_term_d<MODE>(sc * v, sc * acc[i][j], a.beta);
            else local += loss_term_d<MODE>(v, acc[i][j], a.beta);
          } else {
            float pn, pp;
            phi_d<MODE>(v, acc[i][j], bm2, bm1, pn, pp);
            a.Pn[off] = pn;
            if (MODE != kKL) a.Pp[off] = pp;
            else if (MASK) a.Pp[off] = 1.f;
          }
        }
      }
    }
    if (LOSS || (FILL && a.block_partials)) {
      const double tot = block_sum_d((double)local, red);
      if (tid == 0)
        a.block_partials[((int64_t)b * gridDim.y + blockIdx.y) * (RAGGED ? (unsigned)gx : gridDim.x) + blockIdx.x] = tot;
    }
  } else {
    const int64_t HI = s.h_inner();
    float* out = a.out + (int64_t)split * (BATCH && !RAGGED ? bt.n * bt.p : (int64_t)s.B * s.R * HI);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = m0 + 4 * ty + i;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int jj = l0 + 4 * lt + j;
        if (r < s.R && jj < s.Lin && o < OUT) out[((int64_t)b * s.R + r) * HI + (int64_t)o * s.Lin + jj] = acc[i][j];
      }
    }
  }
}

// ---- wgrad: out[split][c, r, (t1, t2), t] = sum over this split's lines (b, j1, j2) and l of
//                                              G[b, c, (j1 + t1, j2 + t2), l] H[b, r, (j1, j2), l - t]
// A block owns MT channels x NCOL columns.  A column is (outer offset, component, offset t): TP = roundup(T, 4) <= 64 offsets
// of NR components (their H windows are staged once per line) for each of NO outer offsets (each with its own G tile).
// grid (t tiles * r groups * outer-offset groups, c tiles, nsplit), 256 threads.
// BATCH: grid z is (problem, split) from z0 on, problem-major, over bt.n problems; problem `prob` reads Gm + prob bt.g and
// H + prob bt.f and writes out[split][prob] (bt.p floats per problem), summing its own lines in the single problem's splits.
// RAGGED (BATCH, bt.rag; s the padded shape): problem `prob` reads its ratio tile in its own compact layout at Gm +
// rag[prob].pn and H in its padded layout, up to its own lengths rag[prob].rows / .lin along the sliding axis, and writes
// its split slabs at out + rag[prob].part, split after split (the plan and the splits do not depend on the length).

template <int MT, bool BATCH = false, bool RAGGED = false>
__global__ void __launch_bounds__(256)
nmfd_wgrad_kernel(NmfdShape s, const float* __restrict__ Gm, const float* __restrict__ H, float* __restrict__ out,
                  int nsplit, WgradPlan p, Batch bt, int64_t z0) {
  static_assert(!RAGGED || BATCH, "RAGGED: a batch");
  using G = Geo<MT>;
  const int hpitch = s.Lin;                   // H's padded pitch (RAGGED: s then holds the problem's lengths)
  if constexpr (RAGGED) {
    const RaggedProblem& rp = bt.rag[(z0 + blockIdx.z) / nsplit];
    s.L = (int)rp.rows; s.Lin = rp.lin;
  }
  __shared__ __align__(16) float Gs[G::NTO * kTK * G::PAD];      // Gs[oo][ll][c]
  __shared__ float Hs[G::HS];
  const int tid = threadIdx.x, tx = tid % G::TX, ty = tid / G::TX;
  const int TP = p.tp, NR = p.nr, NO = p.no;
  const int WIN = TP + kTK;
  const int col = 4 * tx;                                 // TP is a multiple of 4: a thread's 4 columns share (oo, rl)
  const int oo = col / (NR * TP), rl = (col - oo * NR * TP) / TP, tl = col - (oo * NR + rl) * TP;
  const int nouter = s.T1 * s.T2;
  int bx = blockIdx.x;
  const int og = bx % p.nog; bx /= p.nog;
  const int rg = bx % p.nrg;
  const int t0 = (bx / p.nrg) * TP;
  const int c0 = blockIdx.y * MT;
  const int r = rg * NR + rl, to = og * NO + oo;
  const bool live = oo < NO && to < nouter && r < s.R;
  const int J1 = s.J1(), J2 = s.J2();
  const int64_t VI = s.v_inner();
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  // the lines are split over blockIdx.z: more blocks than the output tiles alone give, and shorter fp32 sums
  // 64-bit: create admits up to 2^31 - 1 lines, and the rounded-up split end may pass that
  const int64_t nlines = (int64_t)s.B * J1 * J2, lps = (nlines + nsplit - 1) / nsplit;
  if constexpr (BATCH) {
    const int64_t z = z0 + blockIdx.z, prob = z / nsplit, split = z - prob * nsplit;
    if (batch_skips(bt.active, prob)) return;
    H += prob * bt.f;
    if constexpr (RAGGED) {
      Gm += bt.rag[prob].pn;
      out += bt.rag[prob].part + split * bt.p;
    } else {
      Gm += prob * bt.g;
      out += (split * bt.n + prob) * bt.p;
    }
    z0 = split;                 // from here on: this block's split
  }
  const int64_t zs = BATCH ? z0 : (int64_t)blockIdx.z;
  const int64_t line0 = zs * lps, line1 = min(nlines, line0 + lps);
  if (!BATCH) out += zs * s.C * s.R * s.w_inner();
  for (int64_t bo = line0; bo < line1; ++bo) {            // every H line (b, j1, j2) meets the G lines (b, j1 + t1, j2 + t2)
    const int b = (int)(bo / (J1 * J2)), jo = (int)(bo - (int64_t)b * (J1 * J2));
    const int j1 = jo / J2, j2 = jo - j1 * J2;
    const float* Hb = H + ((int64_t)b * s.R * J1 * J2 + jo) * hpitch;          // + r * J1 * J2 * hpitch per component
    const float* Gb = Gm + (int64_t)b * s.C * VI;
    for (int l0 = 0; l0 < s.L; l0 += kTK) {
      __syncthreads();
      for (int idx = tid; idx < NO * MT * kTK; idx += 256) {
        const int q = idx / kTK, ll = idx - q * kTK;
        const int o2 = q / MT, c = q - o2 * MT;
        const int tq = og * NO + o2;
        float g = 0.f;
        if (tq < nouter && c0 + c < s.C && l0 + ll < s.L) {
          const int t1 = tq / s.T2, t2 = tq - t1 * s.T2;
          g = Gb[(int64_t)(c0 + c) * VI + ((int64_t)(j1 + t1) * s.X2 + (j2 + t2)) * s.L + l0 + ll];
        }
        Gs[(o2 * kTK + ll) * G::PAD + c] = g;
      }
      for (int idx = tid; idx < NR * (WIN - 1); idx += 256) {
        const int rr = idx / (WIN - 1), i = idx - rr * (WIN - 1);
        const int src = l0 - t0 - (TP - 1) + i;           // window index of (ll, tj): ll - tj + TP - 1
        float h = 0.f;
        if (rg * NR + rr < s.R && src >= 0 && src < s.Lin) h = Hb[(int64_t)(rg * NR + rr) * J1 * J2 * hpitch + src];
        Hs[rr * WIN + i] = h;
      }
      __syncthreads();
      if (live) {
        const float* hs = Hs + rl * WIN + (TP - 1 - tl);
        const float* gs = Gs + oo * kTK * G::PAD + 4 * ty;
        const int lmax = min(kTK, s.L - l0);
        float h[4];
        h[0] = hs[-1]; h[1] = hs[-2]; h[2] = hs[-3];       // tl <= TP - 4: the indices are >= 0
#pragma unroll 8
        for (int ll = 0; ll < lmax; ++ll) {
          h[3] = h[2]; h[2] = h[1]; h[1] = h[0];
          h[0] = hs[ll];
          const float4 av4 = *reinterpret_cast<const float4*>(&gs[ll * G::PAD]);
          const float av[4] = {av4.x, av4.y, av4.z, av4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], h[j], acc[i][j]);
        }
      }
    }
  }
  if (!live) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + 4 * ty + i;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int t = t0 + tl + j;
      if (c < s.C && t < s.T) out[(((int64_t)c * s.R + r) * nouter + to) * s.T + t] = acc[i][j];
    }
  }
}

inline int row_tile(int n) { return n <= 4 ? 4 : n <= 8 ? 8 : n <= 16 ? 16 : n <= 32 ? 32 : 64; }
inline int xt_of(int mt) { return (256 / (mt / 4)) / 16; }

inline WgradPlan wgrad_plan(const NmfdShape& s) {
  WgradPlan p;
  p.mt = row_tile(s.C);
  const int ncol = 4 * (256 / (p.mt / 4));
  const int nto = p.mt <= 16 ? 8 : 1;
  p.tp = (int)round_up(s.T < 64 ? s.T : 64, 4);
  p.nr = ncol / p.tp;
  if (p.nr > s.R) p.nr = s.R;
  if (p.nr < 1) p.nr = 1;
  p.no = 1;
  if (p.nr == s.R) {                                       // every component fits: fill the block with outer offsets
    p.no = ncol / (p.nr * p.tp);
    if (p.no > nto) p.no = nto;
    if (p.no > s.T1 * s.T2) p.no = s.T1 * s.T2;
    if (p.no < 1) p.no = 1;
  }
  p.ntt = (int)ceil_div(s.T, p.tp);
  p.nrg = (int)ceil_div(s.R, p.nr);
  p.nog = (int)ceil_div(s.T1 * s.T2, p.no);
  return p;
}

// grid of one launch of the sliding kernel; z = the batch elements per launch (nmfd_batch_slice)
Grid3 slide_grid(const NmfdShape& s, bool fwd, int mt, int M, int nsplit) {
  const int64_t out_lines = fwd ? (int64_t)s.X1 * s.X2 : (int64_t)s.J1() * s.J2();
  const int64_t lout = fwd ? s.L : s.Lin;
  return Grid3{ceil_div(lout, kLT) * ceil_div(out_lines, xt_of(mt)), ceil_div(M, mt) * nsplit, nmfd_batch_slice(s.B)};
}

dim3 dim3_of(const Grid3& g) { return dim3((unsigned)g.x, (unsigned)g.y, (unsigned)g.z); }


// TV: the target's element type (FWD only; the dgrad pass reads no V and always takes float)
template <int MT, bool FWD, typename TV, typename SEL, bool BATCH, bool RAGGED>
void launch_slide(const NmfdShape& s, const SlideArgs& a, const Batch& bt, int mode, bool loss, dim3 grid, cudaStream_t st) {
  if (!FWD) {
    nmfd_slide_kernel<MT, false, kKL, false, float, NoSel, BATCH, RAGGED><<<grid, 256, 0, st>>>(s, a, bt);
    return;
  }
#define NMFD_GO(M)                                                                                          \
  if (loss) nmfd_slide_kernel<MT, true, M, true, TV, SEL, BATCH, RAGGED><<<grid, 256, 0, st>>>(s, a, bt);   \
  else nmfd_slide_kernel<MT, true, M, false, TV, SEL, BATCH, RAGGED><<<grid, 256, 0, st>>>(s, a, bt);
  if constexpr (std::is_same<TV, float>::value && std::is_same<SEL, uint8_t>::value && !BATCH && !RAGGED) {
    if (mode == kPlcaFill) { nmfd_slide_kernel<MT, true, kPlcaFill, false, TV, SEL, false><<<grid, 256, 0, st>>>(s, a, bt); return; }
  }
  switch (mode) {
    case kKL: NMFD_GO(kKL); break;
    case kEU: NMFD_GO(kEU); break;
    case kIS: NMFD_GO(kIS); break;
    default: NMFD_GO(kGeneric); break;
  }
#undef NMFD_GO
}

template <bool FWD, typename TV, typename SEL, bool BATCH, bool RAGGED = false>
void dispatch_slide(int mt, const NmfdShape& s, const SlideArgs& a, const Batch& bt, int mode, bool loss, dim3 grid,
                    cudaStream_t st) {
  switch (mt) {
    case 4: launch_slide<4, FWD, TV, SEL, BATCH, RAGGED>(s, a, bt, mode, loss, grid, st); break;
    case 8: launch_slide<8, FWD, TV, SEL, BATCH, RAGGED>(s, a, bt, mode, loss, grid, st); break;
    case 16: launch_slide<16, FWD, TV, SEL, BATCH, RAGGED>(s, a, bt, mode, loss, grid, st); break;
    case 32: launch_slide<32, FWD, TV, SEL, BATCH, RAGGED>(s, a, bt, mode, loss, grid, st); break;
    default: launch_slide<64, FWD, TV, SEL, BATCH, RAGGED>(s, a, bt, mode, loss, grid, st); break;
  }
}

// one launch of the sliding kernel per slice of at most kMaxGridYZ lines: s.B batch elements, or a batch's bt.n x s.B (a ragged
// batch's grid sized for its padded shape, a.nsplit its largest dgrad split count)
template <bool FWD, typename TV = float, typename SEL = NoSel>
int launch_slices(int mt, const NmfdShape& s, SlideArgs a, const Batch& bt, int mode, bool loss, cudaStream_t st) {
  const int64_t lines = s.B * bt.n;
  Grid3 g = slide_grid(s, FWD, mt, a.M, a.nsplit);
  g.z = nmfd_batch_slice(lines);
  for (int64_t b0 = 0; b0 < lines; b0 += g.z) {
    a.b0 = (int)b0;
    dim3 grid = dim3_of(g);
    grid.z = (unsigned)std::min<int64_t>(g.z, lines - b0);
    bool batched = false;                 // a batch runs the BATCH instantiations (no selector); one problem the others
    if constexpr (std::is_same<SEL, NoSel>::value) batched = bt.n > 1 || bt.active || bt.scale || bt.rag;
    if (batched && bt.rag) {
      if constexpr (std::is_same<SEL, NoSel>::value) dispatch_slide<FWD, TV, SEL, true, true>(mt, s, a, bt, mode, loss, grid, st);
    } else if (batched) {
      if constexpr (std::is_same<SEL, NoSel>::value) dispatch_slide<FWD, TV, SEL, true>(mt, s, a, bt, mode, loss, grid, st);
    } else {
      dispatch_slide<FWD, TV, SEL, false>(mt, s, a, bt, mode, loss, grid, st);
    }
    NMF_LAUNCH_CHECK();
  }
  return 0;
}

// The per-problem offsets of a batch of problems of shape s from the caller's bt.n, bt.v and bt.active: A = W, X = H or G,
// P = Pn / Pp (FWD) or the dgrad partials of one split
Batch slide_batch(const NmfdShape& s, bool fwd, const Batch& bt) {
  Batch b = bt;
  b.f = (int64_t)s.C * s.R * s.w_inner();
  const int64_t vol = (int64_t)s.B * s.C * s.v_inner(), hvol = (int64_t)s.B * s.R * s.h_inner();
  b.g = fwd ? hvol : vol;
  b.p = fwd ? vol : hvol;
  return b;
}

}  // namespace

int64_t nmfd_max_blocks(const NmfdShape& s) {
  const Grid3 g = slide_grid(s, true, row_tile(s.C), s.C, 1);
  return g.x * g.y * s.B;
}

int nmfd_recon_phi(const NmfdShape& s, const void* V, int vdtype, const float* W, const float* H, double beta, float* Pn,
                   float* Pp, double* loss_blocks, int max_blocks, double* loss_dev, cudaStream_t st, CellSel M,
                   const Batch& bt) {
  const int mt = row_tile(s.C);
  const int nblocks = (int)nmfd_max_blocks(s);          // per problem; create bounds it (nmfd_shape_of)
  const bool loss = loss_blocks != nullptr;
  if (bt.n < 1 || ((bt.n > 1 || bt.rag) && M)) { set_error("nmfd_recon_phi: a batch takes no selector"); return 1; }
  if (bt.rag && bt.scale) { set_error("nmfd_recon_phi: a ragged batch takes no scale"); return 1; }
  // a ragged batch's buffer holds its problems' own partials, as its create sized it
  if (loss && !bt.rag && (double)nblocks * (double)bt.n > (double)max_blocks) {
    set_error("nmfd loss: partial buffer too small");
    return 1;
  }
  SlideArgs a{};
  a.A = W; a.X = H; a.M = s.C; a.K = s.R; a.sm = (int64_t)s.R * s.w_inner(); a.sk = s.w_inner(); a.nsplit = 1;
  a.V = V; a.beta = (float)beta; a.Pn = Pn; a.Pp = Pp; a.block_partials = loss_blocks; a.out = nullptr; a.mask = M.p;
  if (int rc = with_vtype(V, vdtype, [&](auto Vt) {
        return with_sel(M, [&](auto Mk) {
          return launch_slices<true, vtype_t<decltype(Vt)>, sel_t<decltype(Mk)>>(mt, s, a, slide_batch(s, true, bt),
                                                                                  beta_mode(beta), loss, st);
        });
      }))
    return rc;
  if (loss) return sum_partials(loss_blocks, nblocks, loss_dev, st, bt.n, bt.active, bt.rag);
  return 0;
}

int nmfd_plca_fill(const NmfdShape& s, const float* V, const float* W, const float* H, float* Pn, float* Pp,
                   const uint8_t* M, double* part, int max_blocks, double* qobs_dev, cudaStream_t st) {
  const int mt = row_tile(s.C);
  const int nblocks = (int)nmfd_max_blocks(s);
  if (!M) { set_error("nmfd_plca_fill: needs the mask"); return 1; }
  if (qobs_dev && (!part || nblocks > max_blocks)) { set_error("nmfd_plca_fill: partial buffer too small"); return 1; }
  SlideArgs a{};
  a.A = W; a.X = H; a.M = s.C; a.K = s.R; a.sm = (int64_t)s.R * s.w_inner(); a.sk = s.w_inner(); a.nsplit = 1;
  a.V = V; a.beta = 1.f; a.Pn = Pn; a.Pp = Pp; a.block_partials = qobs_dev ? part : nullptr; a.out = nullptr; a.mask = M;
  if (int rc = launch_slices<true, float, uint8_t>(mt, s, a, slide_batch(s, true, Batch{}), kPlcaFill, false, st)) return rc;
  if (qobs_dev) return sum_partials(part, nblocks, qobs_dev, st);
  return 0;
}

int nmfd_wgrad_nsplit(const NmfdShape& s) {
  const WgradPlan p = wgrad_plan(s);
  const int64_t tiles = (int64_t)p.ntt * p.nrg * p.nog * ceil_div(s.C, p.mt);
  int64_t ns = ceil_div(132 * 4, tiles);
  const int64_t nlines = (int64_t)s.B * s.J1() * s.J2();
  if (ns > nlines) ns = nlines;
  if (ns > 64) ns = 64;
  if (ns < 1) ns = 1;
  return (int)ns;
}

int nmfd_wgrad(const NmfdShape& s, const float* G, const float* H, float* out, int nsplit, cudaStream_t st, const Batch& bt) {
  const WgradPlan p = wgrad_plan(s);
  const int ncol = 4 * (256 / (p.mt / 4));
  if (p.nr * (p.tp + kTK) > (ncol / 4) * (4 + kTK)) { set_error("nmfd_wgrad: internal tile plan exceeds shared memory"); return 1; }
  if (bt.n < 1) { set_error("nmfd_wgrad: bad problem count"); return 1; }
  Grid3 g = wgrad_grid(s, p, nsplit);
  const bool batched = bt.n > 1 || bt.active || bt.rag;
  Batch b = bt;                           // a batch: problem after problem on grid z, sliced at kMaxGridYZ
  b.f = (int64_t)s.B * s.R * s.h_inner(); b.g = (int64_t)s.B * s.C * s.v_inner(); b.p = (int64_t)s.C * s.R * s.w_inner();
  const int64_t zall = g.z * bt.n;
  for (int64_t z0 = 0; z0 < zall; z0 += kMaxGridYZ) {
    dim3 grid = dim3_of(Grid3{g.x, g.y, std::min<int64_t>(zall - z0, kMaxGridYZ)});
#define NMFD_WGRAD(MT)                                                                           \
  if (bt.rag) nmfd_wgrad_kernel<MT, true, true><<<grid, 256, 0, st>>>(s, G, H, out, nsplit, p, b, z0); \
  else if (batched) nmfd_wgrad_kernel<MT, true><<<grid, 256, 0, st>>>(s, G, H, out, nsplit, p, b, z0); \
  else nmfd_wgrad_kernel<MT><<<grid, 256, 0, st>>>(s, G, H, out, nsplit, p, b, 0);
    switch (p.mt) {
      case 4: NMFD_WGRAD(4); break;
      case 8: NMFD_WGRAD(8); break;
      case 16: NMFD_WGRAD(16); break;
      case 32: NMFD_WGRAD(32); break;
      default: NMFD_WGRAD(64); break;
    }
#undef NMFD_WGRAD
    NMF_LAUNCH_CHECK();
  }
  return 0;
}

int nmfd_dgrad_nsplit(const NmfdShape& s) {
  const Grid3 g = slide_grid(s, false, row_tile(s.R), s.R, 1);
  const int64_t tiles = g.x * g.y * s.B;
  int64_t ns = ceil_div(132 * 4, tiles);
  if (ns > s.C) ns = s.C;
  if (ns > 64) ns = 64;
  if (ns < 1) ns = 1;
  return (int)ns;
}

Grid3 wgrad_grid(const NmfdShape& s, const WgradPlan& p, int nsplit) {
  return Grid3{(int64_t)p.ntt * p.nrg * p.nog, ceil_div(s.C, p.mt), nsplit};
}

void nmfd_plan(const NmfdShape& s, NmfdPlan* p) {
  p->recon_mt = row_tile(s.C);
  p->recon_grid = slide_grid(s, true, p->recon_mt, s.C, 1);
  p->dgrad_mt = row_tile(s.R);
  p->dgrad_nsplit = nmfd_dgrad_nsplit(s);
  p->dgrad_grid = slide_grid(s, false, p->dgrad_mt, s.R, p->dgrad_nsplit);
  p->wgrad = wgrad_plan(s);
  p->wgrad_nsplit = nmfd_wgrad_nsplit(s);
  p->wgrad_grid = wgrad_grid(s, p->wgrad, p->wgrad_nsplit);
}

int nmfd_dgrad(const NmfdShape& s, const float* G, const float* W, float* out, int nsplit, cudaStream_t st, const Batch& bt) {
  if (s.R > 256) { set_error("nmfd_dgrad: rank must be <= 256"); return 1; }
  if (bt.n < 1) { set_error("nmfd_dgrad: bad problem count"); return 1; }
  const int mt = row_tile(s.R);
  SlideArgs a{};
  a.A = W; a.X = G; a.M = s.R; a.K = s.C; a.sm = s.w_inner(); a.sk = (int64_t)s.R * s.w_inner(); a.nsplit = nsplit;
  a.out = out;
  return launch_slices<false>(mt, s, a, slide_batch(s, false, bt), 0, false, st);
}

}  // namespace nmfb200
