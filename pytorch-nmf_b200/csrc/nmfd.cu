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
// grid (line tiles * line groups, row tiles * nsplit, B), 256 threads
struct SlideArgs {
  const float* A;            // W
  const float* X;            // H (FWD) or G
  int M, K;                  // rows of the output, size of the reduced dimension
  int64_t sm, sk;            // strides of A over m and k (elements); the offset (t1, t2, t) is contiguous
  int nsplit;                // !FWD: splits of k
  const float* V; float beta; float* Pn; float* Pp; double* block_partials;     // FWD epilogue
  float* out;                // !FWD: [split][B][R][h_inner]
};

template <int MT, bool FWD, int MODE, bool LOSS>
__global__ void __launch_bounds__(256)
nmfd_slide_kernel(NmfdShape s, SlideArgs a) {
  using G = Geo<MT>;
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
  const int b = blockIdx.z;
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
              x = a.X[((((int64_t)b * a.K + k) * J1 + j1) * J2 + j2) * s.Lin + src];
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
          const float v = a.V[off];
          if (LOSS) {
            local += loss_term_d<MODE>(v, acc[i][j], a.beta);
          } else {
            float pn, pp;
            phi_d<MODE>(v, acc[i][j], bm2, bm1, pn, pp);
            a.Pn[off] = pn;
            if (MODE != kKL) a.Pp[off] = pp;
          }
        }
      }
    }
    if (LOSS) {
      const double tot = block_sum_d((double)local, red);
      if (tid == 0)
        a.block_partials[((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = tot;
    }
  } else {
    const int64_t HI = s.h_inner();
    float* out = a.out + (int64_t)split * s.B * s.R * HI;
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

template <int MT>
__global__ void __launch_bounds__(256)
nmfd_wgrad_kernel(NmfdShape s, const float* __restrict__ Gm, const float* __restrict__ H, float* __restrict__ out,
                  int nsplit, WgradPlan p) {
  using G = Geo<MT>;
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
  const int nlines = s.B * J1 * J2, lps = (nlines + nsplit - 1) / nsplit;
  const int line0 = blockIdx.z * lps, line1 = min(nlines, line0 + lps);
  out += (int64_t)blockIdx.z * s.C * s.R * s.w_inner();
  for (int bo = line0; bo < line1; ++bo) {                // every H line (b, j1, j2) meets the G lines (b, j1 + t1, j2 + t2)
    const int b = bo / (J1 * J2), jo = bo - b * (J1 * J2);
    const int j1 = jo / J2, j2 = jo - j1 * J2;
    const float* Hb = H + ((int64_t)b * s.R * J1 * J2 + jo) * s.Lin;           // + r * J1 * J2 * Lin per component
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
        if (rg * NR + rr < s.R && src >= 0 && src < s.Lin) h = Hb[(int64_t)(rg * NR + rr) * J1 * J2 * s.Lin + src];
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

dim3 slide_grid(const NmfdShape& s, bool fwd, int mt, int M, int nsplit) {
  const int64_t out_lines = fwd ? (int64_t)s.X1 * s.X2 : (int64_t)s.J1() * s.J2();
  const int64_t lout = fwd ? s.L : s.Lin;
  return dim3((unsigned)(ceil_div(lout, kLT) * ceil_div(out_lines, xt_of(mt))), (unsigned)(ceil_div(M, mt) * nsplit),
              (unsigned)s.B);
}

template <int MT, bool FWD>
void launch_slide(const NmfdShape& s, const SlideArgs& a, int mode, bool loss, dim3 grid, cudaStream_t st) {
  if (!FWD) { nmfd_slide_kernel<MT, false, kKL, false><<<grid, 256, 0, st>>>(s, a); return; }
#define NMFD_GO(M)                                                              \
  if (loss) nmfd_slide_kernel<MT, true, M, true><<<grid, 256, 0, st>>>(s, a);   \
  else nmfd_slide_kernel<MT, true, M, false><<<grid, 256, 0, st>>>(s, a);
  switch (mode) {
    case kKL: NMFD_GO(kKL); break;
    case kEU: NMFD_GO(kEU); break;
    case kIS: NMFD_GO(kIS); break;
    default: NMFD_GO(kGeneric); break;
  }
#undef NMFD_GO
}

template <bool FWD>
void dispatch_slide(int mt, const NmfdShape& s, const SlideArgs& a, int mode, bool loss, dim3 grid, cudaStream_t st) {
  switch (mt) {
    case 4: launch_slide<4, FWD>(s, a, mode, loss, grid, st); break;
    case 8: launch_slide<8, FWD>(s, a, mode, loss, grid, st); break;
    case 16: launch_slide<16, FWD>(s, a, mode, loss, grid, st); break;
    case 32: launch_slide<32, FWD>(s, a, mode, loss, grid, st); break;
    default: launch_slide<64, FWD>(s, a, mode, loss, grid, st); break;
  }
}

}  // namespace

int nmfd_max_blocks(const NmfdShape& s) {
  const dim3 g = slide_grid(s, true, row_tile(s.C), s.C, 1);
  return (int)((int64_t)g.x * g.y * g.z);
}

int nmfd_recon_phi(const NmfdShape& s, const float* V, const float* W, const float* H, double beta, float* Pn,
                   float* Pp, double* loss_blocks, int max_blocks, double* loss_dev, cudaStream_t st) {
  const int mt = row_tile(s.C);
  const dim3 grid = slide_grid(s, true, mt, s.C, 1);
  const int nblocks = (int)((int64_t)grid.x * grid.y * grid.z);
  const bool loss = loss_blocks != nullptr;
  if (loss && nblocks > max_blocks) { set_error("nmfd loss: partial buffer too small"); return 1; }
  SlideArgs a{};
  a.A = W; a.X = H; a.M = s.C; a.K = s.R; a.sm = (int64_t)s.R * s.w_inner(); a.sk = s.w_inner(); a.nsplit = 1;
  a.V = V; a.beta = (float)beta; a.Pn = Pn; a.Pp = Pp; a.block_partials = loss_blocks; a.out = nullptr;
  dispatch_slide<true>(mt, s, a, beta_mode(beta), loss, grid, st);
  NMF_LAUNCH_CHECK();
  if (loss) return sum_partials(loss_blocks, nblocks, loss_dev, st);
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

int nmfd_wgrad(const NmfdShape& s, const float* G, const float* H, float* out, int nsplit, cudaStream_t st) {
  const WgradPlan p = wgrad_plan(s);
  const int ncol = 4 * (256 / (p.mt / 4));
  if (p.nr * (p.tp + kTK) > (ncol / 4) * (4 + kTK)) { set_error("nmfd_wgrad: internal tile plan exceeds shared memory"); return 1; }
  dim3 grid((unsigned)((int64_t)p.ntt * p.nrg * p.nog), (unsigned)ceil_div(s.C, p.mt), (unsigned)nsplit);
  switch (p.mt) {
    case 4: nmfd_wgrad_kernel<4><<<grid, 256, 0, st>>>(s, G, H, out, nsplit, p); break;
    case 8: nmfd_wgrad_kernel<8><<<grid, 256, 0, st>>>(s, G, H, out, nsplit, p); break;
    case 16: nmfd_wgrad_kernel<16><<<grid, 256, 0, st>>>(s, G, H, out, nsplit, p); break;
    case 32: nmfd_wgrad_kernel<32><<<grid, 256, 0, st>>>(s, G, H, out, nsplit, p); break;
    default: nmfd_wgrad_kernel<64><<<grid, 256, 0, st>>>(s, G, H, out, nsplit, p); break;
  }
  NMF_LAUNCH_CHECK();
  return 0;
}

int nmfd_dgrad_nsplit(const NmfdShape& s) {
  const dim3 g = slide_grid(s, false, row_tile(s.R), s.R, 1);
  const int64_t tiles = (int64_t)g.x * g.y * g.z;
  int64_t ns = ceil_div(132 * 4, tiles);
  if (ns > s.C) ns = s.C;
  if (ns > 64) ns = 64;
  if (ns < 1) ns = 1;
  return (int)ns;
}

void nmfd_plan(const NmfdShape& s, NmfdPlan* p) {
  p->recon_mt = row_tile(s.C);
  p->recon_grid = slide_grid(s, true, p->recon_mt, s.C, 1);
  p->dgrad_mt = row_tile(s.R);
  p->dgrad_nsplit = nmfd_dgrad_nsplit(s);
  p->dgrad_grid = slide_grid(s, false, p->dgrad_mt, s.R, p->dgrad_nsplit);
  p->wgrad = wgrad_plan(s);
  p->wgrad_nsplit = nmfd_wgrad_nsplit(s);
}

int nmfd_dgrad(const NmfdShape& s, const float* G, const float* W, float* out, int nsplit, cudaStream_t st) {
  if (s.R > 256) { set_error("nmfd_dgrad: rank must be <= 256"); return 1; }
  const int mt = row_tile(s.R);
  const dim3 grid = slide_grid(s, false, mt, s.R, nsplit);
  SlideArgs a{};
  a.A = W; a.X = G; a.M = s.R; a.K = s.C; a.sm = s.w_inner(); a.sk = (int64_t)s.R * s.w_inner(); a.nsplit = nsplit;
  a.out = out;
  dispatch_slide<false>(mt, s, a, 0, false, grid, st);
  NMF_LAUNCH_CHECK();
  return 0;
}

}  // namespace nmfb200
