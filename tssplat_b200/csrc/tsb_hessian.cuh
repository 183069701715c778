// Assembled Hessian of the geometry energy as 3 x 3 block-CSR (tsb_hessian.cu), used by tsb_capi.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace tsb {

constexpr int kHessT = 128;            // threads (tets) per CTA of the per-tet block kernel
constexpr int kHessRowT = 256;         // threads per CTA of the row gather (one warp per block row)
constexpr int kHessTetFloats = 90;     // per tet: the 10 blocks (k, l), k <= l, of its weighted 12 x 12 Hessian, 9 floats each

struct HessParams {
  const int4 *tets;            // [nele] the caller's vertex ids
  const float *B;              // [9][nele] rest inverse Dm^-1, row-major entries
  const float *op;             // PSD only: [kPsdOpFloats][nele], the projection's operator
  uint8_t *kind;               // [nele] kPsd* (written by the block kernel, or by the projection in PSD mode)
  float *blk;                  // [nele][kHessTetFloats]
  const int32_t *crow;         // [n + 1]
  const float *w;              // [nnzb] M_ij (diagonal: M_ii)
  const int32_t *tblk;         // [16 nele] block index of corner pair (k, l) at 16 t + 4 k + l
  const int32_t *inc_ptr;      // [n + 1]
  const int32_t *inc;          // [4 nele] 4 tet + corner, ascending within a row
  int32_t n, nele;
};

// Exact: activity from the sign of det F (fp64 from the fp32 x), then the barrier or AMIPS Hessian weighted by c2 or c3.
// PSD: the projection's operator (already written to op and kind at x) applied to the 12 unit corner directions.
cudaError_t launch_hessian_blocks(const HessParams &p, const float *x, int order, float c2, float c3, bool psd, cudaStream_t st);
// values[b] = c1 M_ij I + the active tets' blocks of row i, summed in incidence-list order
cudaError_t launch_hessian_gather(const HessParams &p, float c1, float *values, cudaStream_t st);

}  // namespace tsb
