// NMFD, NMF2D and NMF3D on wgmma tensor cores (beta = 1): sliding GEMMs with a Toeplitz operand built in shared memory --
// interface used by capi.cu.  See tc_nmfd.cu.
#pragma once
#include "common.cuh"

namespace nmfb200 {

struct TcNmfdState;

// What the tensor-core path launches for a shape, computed in 64 bits before anything is narrowed: the grids of the operand
// preparation and contraction kernels (recon and dgrad grids per launch: batches beyond grid.z take `slices` launches of at
// most `bslice` elements each, dgrad one launch per 128 components), split counts and buffer pitches.  NMF2D / NMF3D
// (NmfdShape with outer axes): recon's grid.z runs over the B X1 X2 target lines, dgrad's over the B J1 J2 activation lines
// (`hslices` launches of at most `hslice`); for NMFD both are the batch.
struct TcNmfdPlan {
  int64_t Tp, padl, Lp, Lq, Cpad;
  int64_t ws_w, kbs_w, ws_h, kbs_h;       // split-K of wgrad / dgrad: splits, k-blocks per split
  int64_t loss_blocks;                    // recon-loss partials (one per CTA of all slices)
  int64_t nch;                            // 2048-element chunks per H row (prep_h)
  Grid3 prep_w, prep_h, recon, wgrad, dgrad;
  int64_t bslice, slices, dgrad_rblocks;
  int64_t hslice, hslices;
};
// nullptr if every grid and every count the kernels hold in 32 bits fits, else the limit the shape crosses
const char* tc_nmfd_plan(const NmfdShape& d, TcNmfdPlan* p);
bool tc_nmfd_supported(const NmfdShape& d, double beta);
int tc_nmfd_create(TcNmfdState** out, const NmfdShape& d);
void tc_nmfd_destroy(TcNmfdState* s);
// sum(V) for the centring constant kappa (also returned to the host: synchronises `st`); V holds `vdtype` (VDtype) elements
int tc_nmfd_set_target(TcNmfdState* s, const void* V, int vdtype, double* vsum_host, cudaStream_t st);
// brings the fp16 operand copies / column sums / kappa up to date with whichever factor changed since the last call, then
// either writes the centred ratio tile (V / (WH + eps) - kappa) 2^p for the following wgrad / dgrad, or (loss) reduces
// metrics.kl_div
int tc_nmfd_recon(TcNmfdState* s, const void* V, int vdtype, const float* W, const float* H, bool loss, double* loss_dev,
                  cudaStream_t st);
// split-K partial numerators from the ratio tile of the last recon: W side [nsplit][C][R][T], H side [nsplit][B][R][Lin]
// (without the kappa * colsum term, which the ratio stage adds: ApplyArgs::kappa / kappa_vec)
int tc_nmfd_wgrad(TcNmfdState* s, const float** part, int* nsplit, cudaStream_t st);
int tc_nmfd_dgrad(TcNmfdState* s, const float** part, int* nsplit, cudaStream_t st);
// [colsum_W (R) | colsum_H (R)] of the factors as of the last recon (the KL denominators, nmf.py:122-131)
const float* tc_nmfd_colsum(const TcNmfdState* s);
// the ratio stage is about to rewrite W (which = 0) or H (1): slot to atomicMax the new values into (ApplyArgs::absmax_bits)
unsigned int* tc_nmfd_begin_update(TcNmfdState* s, int which, cudaStream_t st);
// the factors were changed outside the library: refresh everything at the next recon
void tc_nmfd_mark_dirty(TcNmfdState* s);
const float* tc_nmfd_kappa(const TcNmfdState* s);
// after a stream synchronise: 1 if an NMFD kernel aborted an internal barrier wait since the last check (record cleared)
int tc_nmfd_check_wait_abort();

}  // namespace nmfb200
