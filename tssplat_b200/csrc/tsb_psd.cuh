// Projected (PSD) Hessian of the per-tet energies on a solver workspace (tsb_psd.cu), used by tsb_capi.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace tsb {

// Per-tet operator, structure of arrays [kPsdOpFloats][nele] (fp32): U (9, row-major), V (9, row-major), A+ (6: 00 11 22
// 12 02 01) and the clamped pair eigenvalues lambda_s+ (3), lambda_a+ (3) for the pairs (0,1), (0,2), (1,2).  120 B/tet.
constexpr int kPsdOpFloats = 30;
constexpr int kPsdT = 256;            // threads per CTA of the product and gather kernels
constexpr int kPsdProjectT = 128;     // threads per CTA of the projection
enum : uint8_t { kPsdInactive = 0, kPsdBarrier = 1, kPsdAmips = 2 };

struct PsdParams {
  const int4 *tets;            // [nele] the caller's vertex ids
  const float *B;              // [9][nele] rest inverse Dm^-1, row-major entries
  float *op;                   // [kPsdOpFloats][nele]
  uint8_t *kind;               // [nele] kPsd*
  float *corner;               // [nele][4][3] the product's corner vectors (weighted)
  const int32_t *inc_ptr;      // [n + 1]
  const int32_t *inc;          // [4 nele] 4 tet + corner, ascending within a vertex
  double *part;                // [n_blocks][2] per-CTA curvature partials (barrier, AMIPS)
  float *curv_m;               // [4] the c1 M product's curvature record
  int32_t nele, n, n_blocks;
};

// The product in the rotated frame, D' = L+(Dh): the clamped scaling block A+ on the diagonal, and for the pairs (0,1),
// (0,2), (1,2) lambda_s+ on the symmetric and lambda_a+ on the antisymmetric part.  op(k) is entry k of the tet's
// operator (18 + 00 11 22 12 02 01 for A+, 24 + pair for lambda_s+, 27 + pair for lambda_a+), read where it is first
// needed.  Shared by the projected product (tsb_psd.cu) and the projected assembly (tsb_hessian.cu).
template <class Op>
__device__ __forceinline__ void psd_frame_product(Op op, const float (&Dh)[3][3], float (&Dp)[3][3]) {
  const float a00 = op(18), a11 = op(19), a22 = op(20), a12 = op(21), a02 = op(22), a01 = op(23);
  Dp[0][0] = a00 * Dh[0][0] + a01 * Dh[1][1] + a02 * Dh[2][2];
  Dp[1][1] = a01 * Dh[0][0] + a11 * Dh[1][1] + a12 * Dh[2][2];
  Dp[2][2] = a02 * Dh[0][0] + a12 * Dh[1][1] + a22 * Dh[2][2];
#pragma unroll
  for (int P = 0; P < 3; ++P) {
    const int i = P == 2 ? 1 : 0, j = P == 0 ? 1 : 2;
    const float s = 0.5f * (Dh[i][j] + Dh[j][i]), a = 0.5f * (Dh[i][j] - Dh[j][i]);
    const float ls = op(24 + P), la = op(27 + P);
    Dp[i][j] = ls * s + la * a;
    Dp[j][i] = ls * s - la * a;
  }
}

// Signed SVD and clamped eigen-system of every tet at x: barrier-active where det F < 0, AMIPS-active where det F > 0 and
// amips != 0.
cudaError_t launch_psd_project(const PsdParams &p, const float *x, int order, int amips, cudaStream_t st);
// hv += c2 P(H_b) v + c3 P(H_a) v (corner kernel, then the per-vertex gather in incidence order); curv: the partials too
cudaError_t launch_psd_apply(const PsdParams &p, const float *v, float c2, float c3, bool curv, float *hv, cudaStream_t st);
// curv_out = {c1 vMv + c2 vHb+v + c3 vHa+v, vMv, vHb+v, vHa+v} from curv_m and the partials
cudaError_t launch_psd_curv(const PsdParams &p, float c1, float c2, float c3, float *curv_out, cudaStream_t st);

}  // namespace tsb
