// Affine coarse space of the per-component Newton-CG preconditioner (tsb_pcg_enable_coarse in include/tssplat_b200.h;
// DESIGN.md section 5, "Affine coarse space").
//
// For x = A X + t every tet has F = A, so E_c = Z^T H Z = sum_t [c2 d2psi_b + c3 d2psi_a](F_t) in F-space, entry
// (3 r + c, 3 s + d) = d2 psi / dF_rc dF_sd; the c1 M term vanishes (M annihilates affine maps).  With the corner form of
// tsb_hessian.cu, d2 psi[dF1, dF2] = al dF1 : dF2 + be ((F : dF1)(C : dF2) + (C : dF1)(F : dF2)) + ga (C : dF1)(C : dF2)
// + sk d2J[dF1, dF2], C = cof F, d2J / dF_rc dF_sd = eps_rsi eps_cdj F_ij.  PSD: column (s, d) is P(H)[e_s e_d^T], the
// projected operator the solve multiplies by.  The tet pass writes one partial of the 45 unique entries per tet chunk
// (fixed order: a shuffle tree per warp, the warps in order); the factor kernel (a warp per component) folds them in
// chunk order.
#include "tsb_coarse.cuh"
#include "tsb_psd.cuh"

namespace tsb {
namespace {

constexpr int kTT = kCoarseTetT;
constexpr int kFT = 128;         // threads per CTA of the factor kernel (warp = component)
constexpr int kCoarseSweeps = 30;

// upper-triangle index of (a, b), a <= b
__host__ __device__ constexpr int upper(int a, int b) { return a * 9 - a * (a - 1) / 2 + (b - a); }

// epsilon_{r s i} for r != s, i = 3 - r - s
__device__ __forceinline__ double eps2(int r, int s) { return s == (r + 1) % 3 ? 1.0 : -1.0; }

// adds v (one entry of this thread's tet) to the warp's partial of entry q
__device__ __forceinline__ void warp_add(double v, int q, double *sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  if ((threadIdx.x & 31) == 0) sh[kCoarseUpper * (threadIdx.x >> 5) + q] = v;
}

// One CTA per tet chunk, thread = tet of the chunk.  PSD: the operators of q's last projection.
template <bool PSD>
__global__ void __launch_bounds__(kTT) coarse_tet_kernel(const CoarseParams co, const float *__restrict__ x, int order, float c2,
                                                         float c3, const PsdParams q) {
  __shared__ double sh[kTT / 32 * kCoarseUpper];
  const int e = co.tchunk[3 * blockIdx.x + 1] + int(threadIdx.x);
  const bool in = e < co.tchunk[3 * blockIdx.x + 2];
  const size_t ne = size_t(co.nele);
  if constexpr (!PSD) {
    double F[3][3] = {}, C[3][3] = {};
    double al = 0.0, be = 0.0, ga = 0.0, sk = 0.0, wt = 0.0;
    if (in) {
      const int4 t4 = co.tets[e];
      const int id[4] = {t4.x, t4.y, t4.z, t4.w};
      float xs[4][3];
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int r = 0; r < 3; ++r) xs[k][r] = x[3 * size_t(id[k]) + r];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          double s = 0.0;
#pragma unroll
          for (int k = 0; k < 3; ++k) s += (double(xs[k + 1][r]) - double(xs[0][r])) * double(co.B[(3 * k + c) * ne + e]);
          F[r][c] = s;
        }
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int r1 = (r + 1) % 3, r2 = (r + 2) % 3, k1 = (c + 1) % 3, k2 = (c + 2) % 3;
          C[r][c] = F[r1][k1] * F[r2][k2] - F[r1][k2] * F[r2][k1];
        }
      const double J = F[0][0] * C[0][0] + F[0][1] * C[0][1] + F[0][2] * C[0][2];
      if (J < 0.0) {              // barrier, the activity rule of the assembled Hessian
        const double m = -J;
        ga = order == 2 ? 2.0 : 12.0 * m * m;
        sk = order == 2 ? -2.0 * m : -4.0 * m * m * m;
        wt = double(c2);
      } else if (J > 0.0 && c3 != 0.f) {
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
    }
#pragma unroll
    for (int a = 0; a < 9; ++a)
#pragma unroll
      for (int b = a; b < 9; ++b) {
        const int r = a / 3, c = a % 3, s = b / 3, d = b % 3;
        const double d2j = (r == s || c == d) ? 0.0 : eps2(r, s) * eps2(c, d) * F[3 - r - s][3 - c - d];
        const double h = (a == b ? al : 0.0) + be * (F[r][c] * C[s][d] + C[r][c] * F[s][d]) + ga * C[r][c] * C[s][d] + sk * d2j;
        warp_add(wt * h, upper(a, b), sh);
      }
  } else {
    float U[3][3] = {}, V[3][3] = {}, Ap[6] = {}, ls[3] = {}, la[3] = {};
    float wt = 0.f;
    if (in) {
      const int t = co.tet[e];
      const uint8_t kind = q.kind[t];
      if (kind != kPsdInactive) {
        const size_t qe = size_t(q.nele);
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          U[k / 3][k % 3] = q.op[k * qe + t];
          V[k / 3][k % 3] = q.op[(9 + k) * qe + t];
        }
#pragma unroll
        for (int k = 0; k < 6; ++k) Ap[k] = q.op[(18 + k) * qe + t];
#pragma unroll
        for (int P = 0; P < 3; ++P) { ls[P] = q.op[(24 + P) * qe + t]; la[P] = q.op[(27 + P) * qe + t]; }
        wt = kind == kPsdBarrier ? c2 : c3;
      }
    }
#pragma unroll
    for (int b = 0; b < 9; ++b) {       // column (s, d): Dh = U^T e_s e_d^T V, entry (r, c) = (U D' V^T)_rc
      const int s = b / 3, d = b % 3;
      float Dh[3][3], Dp[3][3];
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) Dh[i][j] = U[s][i] * V[d][j];
      psd_frame_product([&](int k) { return k < 24 ? Ap[k - 18] : k < 27 ? ls[k - 24] : la[k - 27]; }, Dh, Dp);
#pragma unroll
      for (int a = 0; a <= b; ++a) {
        const int r = a / 3, c = a % 3;
        double h = 0.0;
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
          for (int j = 0; j < 3; ++j) h += double(U[r][i]) * double(Dp[i][j]) * double(V[c][j]);
        warp_add(double(wt) * h, upper(a, b), sh);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x < kCoarseUpper) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kTT / 32; ++w) s += sh[kCoarseUpper * w + threadIdx.x];
    co.epart[kCoarseUpper * size_t(blockIdx.x) + threadIdx.x] = s;
  }
}

// One warp per component, lane k < 9 owning row k of E and of the eigenvectors V (shared memory): E_c from the partials in
// chunk order (E_OUT: written out unshifted), else plus shift_c (S_c (x) I3), cyclic Jacobi in fp64 (each rotation's
// column update lane-parallel, the rows mirrored from the columns), eigenvalues <= floor lambda_max dropped,
// E+ = V diag(1 / lambda) V^T.
template <bool E_OUT>
__global__ void __launch_bounds__(kFT) coarse_factor_kernel(const PcgParams s, const CoarseParams co, const float *__restrict__ shift,
                                                            double *__restrict__ E_out) {
  __shared__ double shA[kFT / 32][81], shV[kFT / 32][81];
  const int w = int(threadIdx.x >> 5), lane = int(threadIdx.x & 31);
  const int c = blockIdx.x * (kFT / 32) + w;
  if (c >= s.n_components) return;
  double *A = shA[w], *V = shV[w];
  for (int q = lane; q < kCoarseUpper; q += 32) {
    double u = 0.0;
    for (int k = co.comp_tchunk[c]; k < co.comp_tchunk[c + 1]; ++k) u += co.epart[kCoarseUpper * size_t(k) + q];
    int a = 0;
    while (upper(a, 8) < q) ++a;           // row of upper-triangle index q
    const int b = a + (q - upper(a, a));
    A[9 * a + b] = u;
    A[9 * b + a] = u;
  }
  __syncwarp();
  if constexpr (E_OUT) {
    for (int k = lane; k < 81; k += 32) E_out[81 * size_t(c) + k] = A[k];
    return;
  } else {
    if (shift && lane < 9) {       // + mu (S (x) I3): entry (3 r + i, 3 r + j) gains mu S_ij
      const double mu = double(shift[c]);
      const double *S6 = co.S + 6 * size_t(c);
      const double Sm[3][3] = {{S6[0], S6[5], S6[4]}, {S6[5], S6[1], S6[3]}, {S6[4], S6[3], S6[2]}};
      const int r = lane / 3, i = lane % 3;
#pragma unroll
      for (int j = 0; j < 3; ++j) A[9 * lane + 3 * r + j] += mu * Sm[i][j];
    }
    if (lane < 9)
      for (int k = 0; k < 9; ++k) V[9 * lane + k] = lane == k ? 1.0 : 0.0;
    __syncwarp();
    double fro = 0.0;
    if (lane < 9)
      for (int k = 0; k < 9; ++k) fro += A[9 * lane + k] * A[9 * lane + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) fro += __shfl_xor_sync(0xFFFFFFFFu, fro, o);
    for (int sweep = 0; sweep < kCoarseSweeps; ++sweep) {
      double off = 0.0;
      if (lane < 9)
        for (int k = lane + 1; k < 9; ++k) off += A[9 * lane + k] * A[9 * lane + k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) off += __shfl_xor_sync(0xFFFFFFFFu, off, o);
      if (!(off > 1e-32 * fro)) break;     // also stops on NaN
      for (int p = 0; p < 8; ++p)
        for (int q = p + 1; q < 9; ++q) {
          const double apq = A[9 * p + q];
          if (apq == 0.0) continue;        // the same value in every lane: the warp stays converged
          const double app = A[9 * p + p], aqq = A[9 * q + q];
          const double theta = (aqq - app) / (2.0 * apq);
          const double t = copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
          const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
          double akp = 0.0, akq = 0.0, vkp = 0.0, vkq = 0.0;
          if (lane < 9) {
            akp = A[9 * lane + p]; akq = A[9 * lane + q];
            vkp = V[9 * lane + p]; vkq = V[9 * lane + q];
          }
          __syncwarp();
          if (lane < 9) {
            V[9 * lane + p] = cs * vkp - sn * vkq;
            V[9 * lane + q] = sn * vkp + cs * vkq;
            if (lane == p) { A[9 * p + p] = app - t * apq; A[9 * p + q] = 0.0; }
            else if (lane == q) { A[9 * q + q] = aqq + t * apq; A[9 * q + p] = 0.0; }
            else {
              const double np = cs * akp - sn * akq, nq = sn * akp + cs * akq;
              A[9 * lane + p] = np; A[9 * p + lane] = np;
              A[9 * lane + q] = nq; A[9 * q + lane] = nq;
            }
          }
          __syncwarp();
        }
    }
    double lmax = -INFINITY;
    for (int k = 0; k < 9; ++k) lmax = fmax(lmax, A[10 * k]);
    if (lane < 9) {
      double inv[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double l = A[10 * k];
        inv[k] = (lmax > 0.0 && l > double(co.floor) * lmax) ? 1.0 / l : 0.0;
      }
      double *out = co.Einv + 81 * size_t(c) + 9 * lane;
      for (int j = 0; j < 9; ++j) {
        double a = 0.0;
#pragma unroll
        for (int k = 0; k < 9; ++k) a += V[9 * lane + k] * inv[k] * V[9 * j + k];
        out[j] = a;
      }
    }
  }
}

// R partials of v, per chunk (thread = entry of the chunk)
__global__ void __launch_bounds__(kPcgChunkVerts) coarse_restrict_kernel(const PcgParams s, const CoarseParams co,
                                                                         const float *__restrict__ v) {
  __shared__ double sh9[kPcgChunkVerts / 32 * 9];
  const int e = s.chunk[3 * blockIdx.x + 1] + int(threadIdx.x);
  double q[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (e < s.chunk[3 * blockIdx.x + 2]) coarse_outer(ld3(v, s.vert[e]), co.Y, e, q);
  block_sum9<kPcgChunkVerts>(q, sh9, co.rpart + 9 * size_t(blockIdx.x));
}

// z = P r + Z E+ R (JACOBI) or z += Z E+ R, R folded by every chunk of the component for itself
template <bool JACOBI>
__global__ void __launch_bounds__(kPcgChunkVerts) coarse_apply_kernel(const PcgParams s, const CoarseParams co,
                                                                      const float *__restrict__ r, float *__restrict__ z) {
  const int c = s.chunk[3 * blockIdx.x];
  double *sh = coarse_shared();
  coarse_fold(co, c, s.comp_chunk[c], s.comp_chunk[c + 1], sh);
  const int e = s.chunk[3 * blockIdx.x + 1] + int(threadIdx.x);
  if (e >= s.chunk[3 * blockIdx.x + 2]) return;
  const int v = s.vert[e];
  const F3 g = coarse_prolong(sh + 9, co.Y, e);
  F3 o = JACOBI ? apply_block(s.pinv, v, ld3(r, v)) : ld3(z, v);
  o.x += g.x; o.y += g.y; o.z += g.z;
  st3(z, v, o);
}

}  // namespace

cudaError_t launch_coarse_tets(const CoarseParams &co, const float *x, int order, float c2, float c3, const PsdParams *q,
                               cudaStream_t st) {
  if (co.n_tchunks == 0) return cudaSuccess;
  if (q) coarse_tet_kernel<true><<<unsigned(co.n_tchunks), kTT, 0, st>>>(co, x, order, c2, c3, *q);
  else coarse_tet_kernel<false><<<unsigned(co.n_tchunks), kTT, 0, st>>>(co, x, order, c2, c3, PsdParams{});
  return cudaGetLastError();
}

cudaError_t launch_coarse_factor(const PcgParams &s, const CoarseParams &co, const float *shift, double *E_out, cudaStream_t st) {
  if (s.n_components == 0) return cudaSuccess;
  const unsigned g = unsigned((s.n_components + kFT / 32 - 1) / (kFT / 32));
  if (E_out) coarse_factor_kernel<true><<<g, kFT, 0, st>>>(s, co, nullptr, E_out);
  else coarse_factor_kernel<false><<<g, kFT, 0, st>>>(s, co, shift, nullptr);
  return cudaGetLastError();
}

cudaError_t launch_coarse_restrict(const PcgParams &s, const CoarseParams &co, const float *v, cudaStream_t st) {
  if (s.n_chunks == 0) return cudaSuccess;
  coarse_restrict_kernel<<<unsigned(s.n_chunks), kPcgChunkVerts, 0, st>>>(s, co, v);
  return cudaGetLastError();
}

cudaError_t launch_coarse_apply(const PcgParams &s, const CoarseParams &co, const float *r, float *z, bool jacobi, cudaStream_t st) {
  if (s.n_chunks == 0) return cudaSuccess;
  if (jacobi) coarse_apply_kernel<true><<<unsigned(s.n_chunks), kPcgChunkVerts, 0, st>>>(s, co, r, z);
  else coarse_apply_kernel<false><<<unsigned(s.n_chunks), kPcgChunkVerts, 0, st>>>(s, co, r, z);
  return cudaGetLastError();
}

}  // namespace tsb
