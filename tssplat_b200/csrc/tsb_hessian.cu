// Assembled Hessian of c1 M + c2 barrier + c3 AMIPS as 3 x 3 block-CSR (tsb_hessian_assemble; DESIGN.md section 5,
// "Assembled Hessian").
//
// With corner vectors a_k (rows of B = Dm^-1 for k = 1..3, a_0 = -sum), dF = sum_k dx_k a_k^T.  For psi(F) with
// g_k = cof(F) a_k = dJ/dx_k, f_k = F a_k and w_kl = F (a_k x a_l), the corner block (k, l) of the tet Hessian is
//   H_kl = al (a_k . a_l) I + be (f_k g_l^T + g_k f_l^T) + ga g_k g_l^T + sk S(w_kl),    S(w)_rs = eps_rst w_t
// (S(w_kl) is the cross-corner block of d2J, zero for k = l):
//   barrier (J < 0, m = -J, phi = m^p):  al = be = 0, ga = phi'' = p (p-1) m^(p-2), sk = phi' = -p m^(p-1)
//   AMIPS (J > 0, psi = I1 / (3 J^(2/3)) - 1, a = 2 / (3 J^(2/3))):  al = a, be = -2a / (3J), ga = 5 a I1 / (9 J^2),
//                                                                     sk = -a I1 / (3J)
// PSD: column (l, s) of P(H) is P(H)[e_s a_l^T]; in the rotated frame Dh = u_s (V^T a_l)^T (u_s = row s of U), and
// entry (k r, l s) = u_r . (D'(Dh) V^T a_k), with D' = L+(Dh) of psd_frame_product (tsb_psd.cuh).
#include "tsb_hessian.cuh"
#include "tsb_psd.cuh"

namespace tsb {
namespace {

// block (k, l), k <= l, within a tet's kHessTetFloats
__host__ __device__ constexpr int tet_block(int k, int l) { return 4 * k - k * (k - 1) / 2 + (l - k); }

// One thread per tet; the CTA's blocks are staged in shared memory and written out contiguously.
template <bool PSD>
__global__ void __launch_bounds__(kHessT) hessian_blocks_kernel(const HessParams p, const float *__restrict__ x, int order,
                                                                 float c2, float c3) {
  __shared__ float sh[kHessT * kHessTetFloats];
  const int t0 = blockIdx.x * kHessT, t = t0 + int(threadIdx.x);
  const size_t ne = size_t(p.nele);
  float *o = sh + threadIdx.x * kHessTetFloats;
  uint8_t kind = kPsdInactive;
  if (t < p.nele) {
    if constexpr (PSD) kind = p.kind[t];
    float a[4][3];            // corner vectors
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int c = 0; c < 3; ++c) a[k + 1][c] = p.B[(3 * k + c) * ne + t];
#pragma unroll
    for (int c = 0; c < 3; ++c) a[0][c] = -(a[1][c] + a[2][c] + a[3][c]);
    if constexpr (!PSD) {
      const int4 q = p.tets[t];
      const int id[4] = {q.x, q.y, q.z, q.w};
      float xs[4][3];
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int r = 0; r < 3; ++r) xs[k][r] = x[3 * size_t(id[k]) + r];
      double F[3][3];       // fp64 from the fp32 x: the edges are exact (near-flat AMIPS tets amplify an edge's rounding)
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          double s = 0.0;
#pragma unroll
          for (int k = 0; k < 3; ++k) s += (double(xs[k + 1][r]) - double(xs[0][r])) * double(a[k + 1][c]);
          F[r][c] = s;
        }
      double C[3][3];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int r1 = (r + 1) % 3, r2 = (r + 2) % 3, k1 = (c + 1) % 3, k2 = (c + 2) % 3;
          C[r][c] = F[r1][k1] * F[r2][k2] - F[r1][k2] * F[r2][k1];
        }
      const double J = F[0][0] * C[0][0] + F[0][1] * C[0][1] + F[0][2] * C[0][2];
      kind = J < 0.0 ? kPsdBarrier : (J > 0.0 && c3 != 0.f ? kPsdAmips : kPsdInactive);
      p.kind[t] = kind;
      if (kind != kPsdInactive) {
        double al, be, ga, sk, wt;
        if (kind == kPsdBarrier) {
          const double m = -J;
          al = 0.0; be = 0.0;
          ga = order == 2 ? 2.0 : 12.0 * m * m;
          sk = order == 2 ? -2.0 * m : -4.0 * m * m * m;
          wt = double(c2);
        } else {
          double tr = 0.0;
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) tr += F[r][c] * F[r][c];
          const double cb = cbrt(J), iJ = 1.0 / J;
          al = 2.0 / (3.0 * cb * cb);
          be = -(2.0 / 3.0) * al * iJ;
          ga = (5.0 / 9.0) * al * tr * iJ * iJ;
          sk = -al * tr * iJ / 3.0;
          wt = double(c3);
        }
        double g[4][3], f[4][3];
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int r = 0; r < 3; ++r) {
            g[k][r] = C[r][0] * a[k][0] + C[r][1] * a[k][1] + C[r][2] * a[k][2];
            f[k][r] = F[r][0] * a[k][0] + F[r][1] * a[k][1] + F[r][2] * a[k][2];
          }
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int l = k; l < 4; ++l) {
            const double bkl = double(a[k][0]) * a[l][0] + double(a[k][1]) * a[l][1] + double(a[k][2]) * a[l][2];
            const double cx[3] = {double(a[k][1]) * a[l][2] - double(a[k][2]) * a[l][1],
                                  double(a[k][2]) * a[l][0] - double(a[k][0]) * a[l][2],
                                  double(a[k][0]) * a[l][1] - double(a[k][1]) * a[l][0]};
            double w[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) w[r] = F[r][0] * cx[0] + F[r][1] * cx[1] + F[r][2] * cx[2];
            float *ob = o + 9 * tet_block(k, l);
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
              for (int s = 0; s < 3; ++s) {
                if (k == l && s < r) continue;          // the diagonal block is written symmetric
                const double S = r == s ? 0.0 : ((s == (r + 1) % 3) ? w[(r + 2) % 3] : -w[(r + 1) % 3]);
                const double h = (r == s ? al * bkl : 0.0) + be * (f[k][r] * g[l][s] + g[k][r] * f[l][s]) +
                                 ga * g[k][r] * g[l][s] + sk * S;
                ob[3 * r + s] = float(wt * h);
                if (k == l) ob[3 * s + r] = float(wt * h);
              }
          }
      }
    } else if (kind != kPsdInactive) {
      float U[3][3], Ap[6], ls[3], la[3], at[4][3];
#pragma unroll
      for (int k = 0; k < 9; ++k) U[k / 3][k % 3] = p.op[k * ne + t];
      {
        float V[3][3];
#pragma unroll
        for (int k = 0; k < 9; ++k) V[k / 3][k % 3] = p.op[(9 + k) * ne + t];
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int j = 0; j < 3; ++j) at[k][j] = V[0][j] * a[k][0] + V[1][j] * a[k][1] + V[2][j] * a[k][2];   // V^T a_k
      }
#pragma unroll
      for (int k = 0; k < 6; ++k) Ap[k] = p.op[(18 + k) * ne + t];      // 00 11 22 12 02 01
#pragma unroll
      for (int P = 0; P < 3; ++P) { ls[P] = p.op[(24 + P) * ne + t]; la[P] = p.op[(27 + P) * ne + t]; }
      const float wt = kind == kPsdBarrier ? c2 : c3;
#pragma unroll
      for (int l = 0; l < 4; ++l)
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          float Dh[3][3], Dp[3][3];
#pragma unroll
          for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) Dh[i][j] = U[s][i] * at[l][j];
          psd_frame_product([&](int k) { return k < 24 ? Ap[k - 18] : k < 27 ? ls[k - 24] : la[k - 27]; }, Dh, Dp);
#pragma unroll
          for (int k = 0; k <= l; ++k) {
            float y[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) y[i] = Dp[i][0] * at[k][0] + Dp[i][1] * at[k][1] + Dp[i][2] * at[k][2];
            float *ob = o + 9 * tet_block(k, l);
#pragma unroll
            for (int r = 0; r < 3; ++r) {
              if (k == l && r > s) continue;          // the diagonal block is written symmetric
              const float h = wt * (U[r][0] * y[0] + U[r][1] * y[1] + U[r][2] * y[2]);
              ob[3 * r + s] = h;
              if (k == l) ob[3 * s + r] = h;
            }
          }
        }
    }
  }
  if (kind == kPsdInactive)
#pragma unroll 1
    for (int q = 0; q < kHessTetFloats; ++q) o[q] = 0.f;
  __syncthreads();
  const int nt = min(kHessT, p.nele - t0);
  float *dst = p.blk + size_t(t0) * kHessTetFloats;
  for (int q = int(threadIdx.x); q < nt * kHessTetFloats; q += kHessT) dst[q] = sh[q];
}

// One warp per block row, one lane per block of the row (32 at a time): c1 M_ij I, then every active tet of the row's
// incidence list in order adds its block (k, l) when the pair's block is the lane's.  Each block takes its tets in
// ascending tet order from either side, so (i, j) and (j, i)^T are bitwise equal.
__global__ void __launch_bounds__(kHessRowT) hessian_gather_kernel(const HessParams p, float c1, float *__restrict__ values) {
  const int i = blockIdx.x * (kHessRowT / 32) + int(threadIdx.x >> 5), lane = int(threadIdx.x & 31);
  if (i >= p.n) return;
  const int b0 = p.crow[i], b1 = p.crow[i + 1], e0 = p.inc_ptr[i], e1 = p.inc_ptr[i + 1];
  for (int base = b0; base < b1; base += 32) {
    const int b = base + lane;
    const float m = b < b1 ? c1 * p.w[b] : 0.f;
    float acc[9] = {m, 0.f, 0.f, 0.f, m, 0.f, 0.f, 0.f, m};
    for (int e = e0; e < e1; ++e) {
      const int c = p.inc[e], t = c >> 2, k = c & 3;
      if (p.kind[t] == kPsdInactive) continue;
      const int4 tb = reinterpret_cast<const int4 *>(p.tblk)[c];
      const int l = tb.x == b ? 0 : (tb.y == b ? 1 : (tb.z == b ? 2 : (tb.w == b ? 3 : -1)));
      if (l < 0) continue;
      const float *src = p.blk + size_t(t) * kHessTetFloats + 9 * tet_block(min(k, l), max(k, l));
      if (k <= l) {
#pragma unroll
        for (int q = 0; q < 9; ++q) acc[q] += src[q];
      } else {
#pragma unroll
        for (int q = 0; q < 9; ++q) acc[q] += src[3 * (q % 3) + q / 3];
      }
    }
    if (b < b1) {
      float *dst = values + 9 * size_t(b);
#pragma unroll
      for (int q = 0; q < 9; ++q) dst[q] = acc[q];
    }
  }
}

}  // namespace

cudaError_t launch_hessian_blocks(const HessParams &p, const float *x, int order, float c2, float c3, bool psd, cudaStream_t st) {
  const unsigned grid = unsigned((p.nele + kHessT - 1) / kHessT);
  if (psd) hessian_blocks_kernel<true><<<grid, kHessT, 0, st>>>(p, x, order, c2, c3);
  else hessian_blocks_kernel<false><<<grid, kHessT, 0, st>>>(p, x, order, c2, c3);
  return cudaGetLastError();
}

cudaError_t launch_hessian_gather(const HessParams &p, float c1, float *values, cudaStream_t st) {
  constexpr int rows = kHessRowT / 32;
  hessian_gather_kernel<<<unsigned((p.n + rows - 1) / rows), kHessRowT, 0, st>>>(p, c1, values);
  return cudaGetLastError();
}

}  // namespace tsb
