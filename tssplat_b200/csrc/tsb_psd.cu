// Projected Newton: the PSD projection of every tet's barrier or AMIPS Hessian and its product with a vector
// (tsb_pcg_enable_psd, tsb_pcg_hvp_psd and the PSD mode of tsb_pcg_solve; DESIGN.md section 5, "Projected Hessian").
//
// Both per-tet energies are isotropic functions of F = Ds B (B = Dm^-1), so with the signed SVD F = U diag(s) V^T (U, V
// proper rotations, sign s_3 = sign det F) the 9 x 9 Hessian in F-space splits into the 3 x 3 scaling block A = d2 Psi /
// ds2 and, per pair (i, j), a symmetric and an antisymmetric twist mode with the closed-form eigenvalues lambda_s and
// lambda_a.  The projection clamps A's eigenvalues and the six pair eigenvalues at 0.  The product in the rotated frame,
// Dh = U^T dF V, D' = L+(Dh), P(H)[dF] = U D' V^T, gives dF : P(H)[dF] = Dh : L+(Dh) >= 0 whatever rounding U and V
// carry, so the stored operator stays PSD in fp32 (A+ up to its own rounding).
#include "tsb_device.cuh"
#include "tsb_jacobi.cuh"
#include "tsb_psd.cuh"

namespace tsb {
namespace {

__device__ __forceinline__ double det3(const double (&F)[3][3]) {
  return F[0][0] * (F[1][1] * F[2][2] - F[1][2] * F[2][1]) - F[0][1] * (F[1][0] * F[2][2] - F[1][2] * F[2][0]) +
         F[0][2] * (F[1][0] * F[2][1] - F[1][1] * F[2][0]);
}

// Symmetric 3x3 (a00 a11 a22 a12 a02 a01) -> eigenvalues ev and eigenvectors as the columns of Q (cyclic Jacobi, the
// rotation and sweep count of the preconditioner blocks).
__device__ __forceinline__ void sym_eig(double a00, double a11, double a22, double a12, double a02, double a01, double (&ev)[3],
                                        double (&Q)[3][3]) {
  double v00 = 1, v01 = 0, v02 = 0, v10 = 0, v11 = 1, v12 = 0, v20 = 0, v21 = 0, v22 = 1;
#pragma unroll 1
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
    if (a01 == 0.0 && a02 == 0.0 && a12 == 0.0) break;
    jacobi_rot(a00, a11, a01, a02, a12, v00, v01, v10, v11, v20, v21);
    jacobi_rot(a00, a22, a02, a01, a12, v00, v02, v10, v12, v20, v22);
    jacobi_rot(a11, a22, a12, a01, a02, v01, v02, v11, v12, v21, v22);
  }
  ev[0] = a00; ev[1] = a11; ev[2] = a22;
  Q[0][0] = v00; Q[0][1] = v01; Q[0][2] = v02;
  Q[1][0] = v10; Q[1][1] = v11; Q[1][2] = v12;
  Q[2][0] = v20; Q[2][1] = v21; Q[2][2] = v22;
}

__device__ __forceinline__ void swap_col(double (&ev)[3], double (&Q)[3][3], int a, int b) {
  double t = ev[a]; ev[a] = ev[b]; ev[b] = t;
#pragma unroll
  for (int r = 0; r < 3; ++r) { t = Q[r][a]; Q[r][a] = Q[r][b]; Q[r][b] = t; }
}

// One-sided (Hestenes) Jacobi rotation of columns p and q of W = F V, and of V with them, that makes w_p and w_q
// orthogonal.  Its angle comes from the columns' own dot products, accurate relative to |w_p| |w_q|; the entries of F^T F
// carry an error of eps s_1^2, which loses the directions of every s_i^2 below that.
__device__ __forceinline__ void hestenes_rot(double (&W)[3][3], double (&V)[3][3], int p, int q) {
  const double al = W[0][p] * W[0][p] + W[1][p] * W[1][p] + W[2][p] * W[2][p];
  const double be = W[0][q] * W[0][q] + W[1][q] * W[1][q] + W[2][q] * W[2][q];
  const double ga = W[0][p] * W[0][q] + W[1][p] * W[1][q] + W[2][p] * W[2][q];
  if (ga == 0.0) return;
  const double theta = (be - al) / (2.0 * ga);
  const double t = copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
  const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    double a = c * W[r][p] - s * W[r][q]; W[r][q] = s * W[r][p] + c * W[r][q]; W[r][p] = a;
    a = c * V[r][p] - s * V[r][q]; V[r][q] = s * V[r][p] + c * V[r][q]; V[r][p] = a;
  }
}

__device__ __forceinline__ void normalize(double (&u)[3]) {
  const double s = 1.0 / sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]);
  u[0] *= s; u[1] *= s; u[2] *= s;
}

// pairs (i, j) and their third index k, in the order of the stored pair eigenvalues
__device__ constexpr int kPi[3] = {0, 0, 1}, kPj[3] = {1, 2, 2}, kPk[3] = {2, 1, 0};

// One thread per tet: F in fp64 from the fp32 edges and B, activity from the sign of det F, signed SVD from the Jacobi
// eigen-decomposition of F^T F refined by one one-sided Jacobi sweep on F V, then the clamped eigen-system.
__global__ void __launch_bounds__(kPsdProjectT) psd_project_kernel(const PsdParams p, const float *__restrict__ x, int order,
                                                                   int amips) {
  const int t = blockIdx.x * kPsdProjectT + int(threadIdx.x);
  if (t >= p.nele) return;
  const size_t ne = size_t(p.nele);
  const int4 q = p.tets[t];
  const int id[4] = {q.x, q.y, q.z, q.w};
  float xs[4][3];
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int r = 0; r < 3; ++r) xs[k][r] = x[3 * size_t(id[k]) + r];
  double F[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      double s = 0.0;
#pragma unroll
      for (int k = 0; k < 3; ++k) s += double(xs[k + 1][r] - xs[0][r]) * double(p.B[(3 * k + c) * ne + t]);
      F[r][c] = s;
    }
  const double J = det3(F);
  const uint8_t kind = J < 0.0 ? kPsdBarrier : (J > 0.0 && amips ? kPsdAmips : kPsdInactive);
  p.kind[t] = kind;
  if (kind == kPsdInactive) return;

  // V and the squared singular values from F^T F, descending, V a proper rotation
  double ev[3], V[3][3];
  {
    double S[3][3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) S[a][b] = F[0][a] * F[0][b] + F[1][a] * F[1][b] + F[2][a] * F[2][b];
    sym_eig(S[0][0], S[1][1], S[2][2], S[1][2], S[0][2], S[0][1], ev, V);
  }
  if (ev[0] < ev[1]) swap_col(ev, V, 0, 1);
  if (ev[1] < ev[2]) swap_col(ev, V, 1, 2);
  if (ev[0] < ev[1]) swap_col(ev, V, 0, 1);
  if (det3(V) < 0.0)
#pragma unroll
    for (int r = 0; r < 3; ++r) V[r][2] = -V[r][2];
  // one one-sided Jacobi sweep on the columns of W = F V refines V where F^T F cannot resolve it (s_2 or s_3 below
  // ~ sqrt(eps) s_1: needles, collapsing planes); then descending column norms and V proper again
  double W[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int i = 0; i < 3; ++i) W[r][i] = F[r][0] * V[0][i] + F[r][1] * V[1][i] + F[r][2] * V[2][i];
  hestenes_rot(W, V, 0, 1);
  hestenes_rot(W, V, 0, 2);
  hestenes_rot(W, V, 1, 2);
  {
    double n2[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) n2[i] = W[0][i] * W[0][i] + W[1][i] * W[1][i] + W[2][i] * W[2][i];
    auto swap_wv = [&](int a, int b) {
      swap_col(n2, V, a, b);
#pragma unroll
      for (int r = 0; r < 3; ++r) { const double t = W[r][a]; W[r][a] = W[r][b]; W[r][b] = t; }
    };
    if (n2[0] < n2[1]) swap_wv(0, 1);
    if (n2[1] < n2[2]) swap_wv(1, 2);
    if (n2[0] < n2[1]) swap_wv(0, 1);
  }
  if (det3(V) < 0.0)
#pragma unroll
    for (int r = 0; r < 3; ++r) { V[r][2] = -V[r][2]; W[r][2] = -W[r][2]; }
  // u_1 = F v_1 / s_1, u_2 = the part of F v_2 orthogonal to u_1, u_3 = u_1 x u_2; s_3 = det F / (s_1 s_2) carries the
  // sign (reflections land in s_3, never in U or V) and stays accurate as s_3 -> 0
  double u[3][3], sg[3];
  double w[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int r = 0; r < 3; ++r) w[i][r] = W[r][i];
  sg[0] = sqrt(w[0][0] * w[0][0] + w[0][1] * w[0][1] + w[0][2] * w[0][2]);
#pragma unroll
  for (int r = 0; r < 3; ++r) u[0][r] = w[0][r] / sg[0];     // sg[0] > 0: det F != 0
  {
    const double pr = u[0][0] * w[1][0] + u[0][1] * w[1][1] + u[0][2] * w[1][2];
#pragma unroll
    for (int r = 0; r < 3; ++r) u[1][r] = w[1][r] - pr * u[0][r];
    sg[1] = sqrt(u[1][0] * u[1][0] + u[1][1] * u[1][1] + u[1][2] * u[1][2]);
    if (!(sg[1] > 1e-150 * sg[0])) {      // not reached for det F != 0 in practice: any unit vector orthogonal to u_1
      const int a = fabs(u[0][0]) < fabs(u[0][1]) ? (fabs(u[0][0]) < fabs(u[0][2]) ? 0 : 2) : (fabs(u[0][1]) < fabs(u[0][2]) ? 1 : 2);
      double e[3] = {0.0, 0.0, 0.0};
      e[a] = 1.0;
      u[1][0] = u[0][1] * e[2] - u[0][2] * e[1];
      u[1][1] = u[0][2] * e[0] - u[0][0] * e[2];
      u[1][2] = u[0][0] * e[1] - u[0][1] * e[0];
    }
    normalize(u[1]);
  }
  u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
  u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
  u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
  sg[2] = J / (sg[0] * sg[1]);

  // A = d2 Psi / ds2 and the pair eigenvalues, cancellation-free (DESIGN.md section 5)
  double A[3][3], ls[3], la[3];
  if (kind == kPsdBarrier) {
    const double m = -J;
    const double d1 = order == 2 ? -2.0 * m : -4.0 * m * m * m;    // phi'(J), phi = (-J)^p
    const double d2 = order == 2 ? 2.0 : 12.0 * m * m;               // phi''(J)
    const double g[3] = {sg[1] * sg[2], sg[0] * sg[2], sg[0] * sg[1]};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) A[i][j] = d2 * g[i] * g[j] + (i == j ? 0.0 : d1 * sg[3 - i - j]);
#pragma unroll
    for (int P = 0; P < 3; ++P) { ls[P] = -d1 * sg[kPk[P]]; la[P] = d1 * sg[kPk[P]]; }
  } else {
    const double cb = cbrt(J), j23 = cb * cb;
    const double al = 2.0 / (3.0 * j23);
    const double ga = 2.0 * (sg[0] * sg[0] + sg[1] * sg[1] + sg[2] * sg[2]) / (9.0 * j23);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j)
        A[i][j] = i == j ? -al / 3.0 + (5.0 / 3.0) * ga / (sg[i] * sg[i])
                         : -(2.0 / 3.0) * al * (sg[i] / sg[j] + sg[j] / sg[i]) + (2.0 / 3.0) * ga / (sg[i] * sg[j]);
#pragma unroll
    for (int P = 0; P < 3; ++P) {
      const double r = ga / (sg[kPi[P]] * sg[kPj[P]]);
      ls[P] = al + r;
      la[P] = al - r;
    }
  }
  double lam[3], Q[3][3];
  sym_eig(A[0][0], A[1][1], A[2][2], A[1][2], A[0][2], A[0][1], lam, Q);
#pragma unroll
  for (int i = 0; i < 3; ++i) lam[i] = fmax(lam[i], 0.0);
  auto ap = [&](int a, int b) { return lam[0] * Q[a][0] * Q[b][0] + lam[1] * Q[a][1] * Q[b][1] + lam[2] * Q[a][2] * Q[b][2]; };
  float o[kPsdOpFloats];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      o[3 * r + i] = float(u[i][r]);
      o[9 + 3 * r + i] = float(V[r][i]);
    }
  o[18] = float(ap(0, 0)); o[19] = float(ap(1, 1)); o[20] = float(ap(2, 2));
  o[21] = float(ap(1, 2)); o[22] = float(ap(0, 2)); o[23] = float(ap(0, 1));
#pragma unroll
  for (int P = 0; P < 3; ++P) {
    o[24 + P] = float(fmax(ls[P], 0.0));
    o[27 + P] = float(fmax(la[P], 0.0));
  }
#pragma unroll
  for (int k = 0; k < kPsdOpFloats; ++k) p.op[k * ne + t] = o[k];
}

// One thread per tet: corner vectors of w P(H_t)[dF] with dF = dDs B, w = c2 (barrier) or c3 (AMIPS); inactive tets
// write nothing (the gather skips them).  CURV: per-CTA fp64 partials of v^T P(H_t) v (unweighted) per term.
template <bool CURV>
__global__ void __launch_bounds__(kPsdT) psd_apply_kernel(const PsdParams p, const float *__restrict__ v, float c2, float c3) {
  const int t = blockIdx.x * kPsdT + int(threadIdx.x);
  const size_t ne = size_t(p.nele);
  const uint8_t kind = t < p.nele ? p.kind[t] : uint8_t(kPsdInactive);
  double qb = 0.0, qa = 0.0;
  if (kind != kPsdInactive) {
    const int4 iq = p.tets[t];
    const int id[4] = {iq.x, iq.y, iq.z, iq.w};
    float vs[4][3], B[3][3], U[3][3], V[3][3];
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int r = 0; r < 3; ++r) vs[k][r] = v[3 * size_t(id[k]) + r];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      B[k / 3][k % 3] = p.B[k * ne + t];
      U[k / 3][k % 3] = p.op[k * ne + t];
      V[k / 3][k % 3] = p.op[(9 + k) * ne + t];
    }
    float dF[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c)
        dF[r][c] = (vs[1][r] - vs[0][r]) * B[0][c] + (vs[2][r] - vs[0][r]) * B[1][c] + (vs[3][r] - vs[0][r]) * B[2][c];
    float T[3][3], Dh[3][3];    // T = U^T dF, Dh = T V
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int c = 0; c < 3; ++c) T[i][c] = U[0][i] * dF[0][c] + U[1][i] * dF[1][c] + U[2][i] * dF[2][c];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) Dh[i][j] = T[i][0] * V[0][j] + T[i][1] * V[1][j] + T[i][2] * V[2][j];
    float Dp[3][3];
    psd_frame_product([&](int k) { return p.op[k * ne + t]; }, Dh, Dp);
    if constexpr (CURV) {
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) q = fmaf(Dh[i][j], Dp[i][j], q);
      (kind == kPsdBarrier ? qb : qa) = double(q);
    }
    float W[3][3], Pm[3][3];    // W = U D', P = W V^T
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int j = 0; j < 3; ++j) W[r][j] = U[r][0] * Dp[0][j] + U[r][1] * Dp[1][j] + U[r][2] * Dp[2][j];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) Pm[r][c] = W[r][0] * V[c][0] + W[r][1] * V[c][1] + W[r][2] * V[c][2];
    const float wt = kind == kPsdBarrier ? c2 : c3;
    float g[12];
#pragma unroll
    for (int r = 0; r < 3; ++r) g[r] = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const float c = wt * (Pm[r][0] * B[k][0] + Pm[r][1] * B[k][1] + Pm[r][2] * B[k][2]);
        g[3 * (k + 1) + r] = c;
        g[r] -= c;
      }
    float4 *dst = reinterpret_cast<float4 *>(p.corner + 12 * size_t(t));
    dst[0] = make_float4(g[0], g[1], g[2], g[3]);
    dst[1] = make_float4(g[4], g[5], g[6], g[7]);
    dst[2] = make_float4(g[8], g[9], g[10], g[11]);
  }
  if constexpr (CURV) {
    __shared__ double sh[kPsdT / 32];
    const double sb = block_sum<kPsdT>(qb, sh);
    if (threadIdx.x == 0) p.part[2 * size_t(blockIdx.x)] = sb;
    const double sa = block_sum<kPsdT>(qa, sh);
    if (threadIdx.x == 0) p.part[2 * size_t(blockIdx.x) + 1] = sa;
  }
}

// One thread per vertex: hv_i += the active corners of its incidence list, summed in list order.
__global__ void __launch_bounds__(kPsdT) psd_gather_kernel(const PsdParams p, float *__restrict__ hv) {
  const int i = blockIdx.x * kPsdT + int(threadIdx.x);
  if (i >= p.n) return;
  float ax = 0.f, ay = 0.f, az = 0.f;
  bool any = false;
  const int e1 = p.inc_ptr[i + 1];
  for (int e = p.inc_ptr[i]; e < e1; ++e) {
    const int c = p.inc[e];
    if (p.kind[c >> 2] == kPsdInactive) continue;
    const float *q = p.corner + 3 * size_t(c);
    ax += q[0]; ay += q[1]; az += q[2];
    any = true;
  }
  if (any) {
    hv[3 * size_t(i)] += ax;
    hv[3 * size_t(i) + 1] += ay;
    hv[3 * size_t(i) + 2] += az;
  }
}

// One CTA: the partials in a fixed order, then the record.
__global__ void __launch_bounds__(kPsdT) psd_curv_kernel(const PsdParams p, float c1, float c2, float c3, float *__restrict__ out) {
  __shared__ double sh[kPsdT / 32];
  double b = 0.0, a = 0.0;
  for (int k = int(threadIdx.x); k < p.n_blocks; k += kPsdT) {
    b += p.part[2 * size_t(k)];
    a += p.part[2 * size_t(k) + 1];
  }
  const double sb = block_sum<kPsdT>(b, sh);
  const double sa = block_sum<kPsdT>(a, sh);
  if (threadIdx.x == 0) {
    const float vmv = p.curv_m[1];
    out[0] = float(double(c1) * double(vmv) + double(c2) * sb + double(c3) * sa);
    out[1] = vmv;
    out[2] = float(sb);
    out[3] = float(sa);
  }
}

}  // namespace

cudaError_t launch_psd_project(const PsdParams &p, const float *x, int order, int amips, cudaStream_t st) {
  psd_project_kernel<<<unsigned((p.nele + kPsdProjectT - 1) / kPsdProjectT), kPsdProjectT, 0, st>>>(p, x, order, amips);
  return cudaGetLastError();
}

cudaError_t launch_psd_apply(const PsdParams &p, const float *v, float c2, float c3, bool curv, float *hv, cudaStream_t st) {
  if (curv) psd_apply_kernel<true><<<unsigned(p.n_blocks), kPsdT, 0, st>>>(p, v, c2, c3);
  else psd_apply_kernel<false><<<unsigned(p.n_blocks), kPsdT, 0, st>>>(p, v, c2, c3);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  psd_gather_kernel<<<unsigned((p.n + kPsdT - 1) / kPsdT), kPsdT, 0, st>>>(p, hv);
  return cudaGetLastError();
}

cudaError_t launch_psd_curv(const PsdParams &p, float c1, float c2, float c3, float *curv_out, cudaStream_t st) {
  psd_curv_kernel<<<1, kPsdT, 0, st>>>(p, c1, c2, c3, curv_out);
  return cudaGetLastError();
}

}  // namespace tsb
