// Per-component (per tet-sphere) block-Jacobi preconditioned truncated CG on the device: the small kernels that run
// between two Hessian-vector products of tsb_pcg_solve (include/tssplat_b200.h; DESIGN.md section 5, "Newton-CG solve").
//
// Spheres share no vertices, so H is block diagonal by component and CG runs independently on every block, all blocks
// in the same launches.  A CTA owns one chunk: <= kPcgChunkVerts consecutive entries of one component's vertex list
// (thread = vertex).  A dot product over a component is two steps: every chunk stores its fp64 partial (a shuffle tree
// and a fixed-order sum over the CTA's warps), and in the next kernel every chunk of the component folds the
// component's partials itself, in chunk order, from a column of the partial table that no CTA of that kernel writes.
// The fold is redundant across the chunks of a component, but it needs no ticket, no atomic and no fence, and every
// chunk gets bitwise the same scalar.  All scalars stay in device memory.
#include "tsb_coarse.cuh"
#include "tsb_device.cuh"
#include "tsb_jacobi.cuh"
#include "tsb_sgs.cuh"
#include "tsb_solver.cuh"

namespace tsb {
namespace {

constexpr int kT = kPcgChunkVerts;   // threads per CTA

// The partial table has three columns per chunk, each with one writing kernel per iteration and read only by the kernel
// after it, so no launch folds a column it also writes: kPHp (pcg_curv_kernel -> pcg_update_kernel; pcg_bdotd_kernel ->
// pcg_record_kernel), kRz and kRr (pcg_init_kernel / pcg_update_kernel -> pcg_dir_kernel).
constexpr int kPartCols = 3, kPHp = 0, kRz = 1, kRr = 2;

// Sum of one column of the partials of chunks [c0, c1) in a fixed order, valid in every thread: lane l of warp 0 adds
// chunks c0 + l, c0 + l + 32, ..., a shuffle tree combines the lanes.
__device__ __forceinline__ double fold(const double *part, int col, int c0, int c1, double *sh) {
  if (threadIdx.x < 32) {
    double a = 0.0;
    for (int k = c0 + int(threadIdx.x); k < c1; k += 32) a += part[kPartCols * size_t(k) + col];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xFFFFFFFFu, a, o);
    if (threadIdx.x == 0) sh[0] = a;
  }
  __syncthreads();
  const double out = sh[0];
  __syncthreads();                                  // sh is reused by the next fold and by block_sum
  return out;
}

// Inverse preconditioner block of vertex v: cyclic Jacobi eigen-decomposition in fp64 registers, eigenvalues clamped
// from below to rel_floor * lambda_max, block inverted; lambda_max <= 0 gives the zero block.  diag == nullptr: the
// identity.  SHIFT: the block is D_v + mu I.
template <bool SHIFT>
__device__ __forceinline__ void block_inverse(const float *__restrict__ diag, int n, int v, float rel_floor, double mu,
                                              float *__restrict__ pinv, float *__restrict__ inv_out) {
  float o[6] = {1.f, 1.f, 1.f, 0.f, 0.f, 0.f};
  if (diag) {
    const float *d0 = diag + 3 * size_t(v), *d1 = diag + 3 * (size_t(n) + size_t(v));
    double a00 = d0[0], a11 = d0[1], a22 = d0[2], a12 = d1[0], a02 = d1[1], a01 = d1[2];
    if (SHIFT) { a00 += mu; a11 += mu; a22 += mu; }
    double v00 = 1, v01 = 0, v02 = 0, v10 = 0, v11 = 1, v12 = 0, v20 = 0, v21 = 0, v22 = 1;
#pragma unroll 1
    for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
      if (a01 == 0.0 && a02 == 0.0 && a12 == 0.0) break;
      jacobi_rot(a00, a11, a01, a02, a12, v00, v01, v10, v11, v20, v21);
      jacobi_rot(a00, a22, a02, a01, a12, v00, v02, v10, v12, v20, v22);
      jacobi_rot(a11, a22, a12, a01, a02, v01, v02, v11, v12, v21, v22);
    }
    const double lmax = fmax(a00, fmax(a11, a22));
    if (lmax > 0.0) {
      const double fl = double(rel_floor) * lmax;
      const double i0 = 1.0 / fmax(a00, fl), i1 = 1.0 / fmax(a11, fl), i2 = 1.0 / fmax(a22, fl);
      o[0] = float(i0 * v00 * v00 + i1 * v01 * v01 + i2 * v02 * v02);
      o[1] = float(i0 * v10 * v10 + i1 * v11 * v11 + i2 * v12 * v12);
      o[2] = float(i0 * v20 * v20 + i1 * v21 * v21 + i2 * v22 * v22);
      o[3] = float(i0 * v10 * v20 + i1 * v11 * v21 + i2 * v12 * v22);
      o[4] = float(i0 * v00 * v20 + i1 * v01 * v21 + i2 * v02 * v22);
      o[5] = float(i0 * v00 * v10 + i1 * v01 * v11 + i2 * v02 * v12);
    } else {
#pragma unroll
      for (int k = 0; k < 6; ++k) o[k] = 0.f;
    }
  }
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    pinv[6 * size_t(v) + k] = o[k];
    if (inv_out) inv_out[6 * size_t(v) + k] = o[k];
  }
}

// Inverse preconditioner block of every vertex (thread = vertex).
__global__ void __launch_bounds__(kT) pcg_blocks_kernel(const float *__restrict__ diag, int n, float rel_floor,
                                                        float *__restrict__ pinv, float *__restrict__ inv_out) {
  const int v = blockIdx.x * kT + int(threadIdx.x);
  if (v >= n) return;
  block_inverse<false>(diag, n, v, rel_floor, 0.0, pinv, inv_out);
}

// The same with the blocks D_v + mu_c I, over the chunk table (thread = vertex of a component, which gives its mu_c);
// CTAs past the chunk table take the orphan vertices, unshifted (their rows of diag are zero: the zero block).
__global__ void __launch_bounds__(kT) pcg_blocks_shift_kernel(const PcgParams s, const float *__restrict__ diag, float rel_floor,
                                                              const float *__restrict__ shift, float *__restrict__ inv_out) {
  int v;
  double mu = 0.0;
  if (int(blockIdx.x) >= s.n_chunks) {
    const int k = (int(blockIdx.x) - s.n_chunks) * kT + int(threadIdx.x);
    if (k >= s.n_orphans) return;
    v = s.orphans[k];
  } else {
    const int e = s.chunk[3 * blockIdx.x + 1] + int(threadIdx.x);
    if (e >= s.chunk[3 * blockIdx.x + 2]) return;
    v = s.vert[e];
    mu = double(shift[s.chunk[3 * blockIdx.x]]);
  }
  block_inverse<true>(diag, s.n, v, rel_floor, mu, s.pinv, inv_out);
}

// r = b, z = P r, d = 0, partials of r.z and r.r.  CTAs past the chunk table zero d on the orphan vertices.  COARSE:
// also the partials of R = Z^T r.  Each kernel is a body instantiated by a __global__ of its own name, so the block-Jacobi
// kernels keep the machine code they had before the coarse variants existed.
template <bool COARSE>
__device__ __forceinline__ void pcg_init_body(const PcgParams &s, const float *__restrict__ b, float *__restrict__ d,
                                              const CoarseParams &co) {
  __shared__ double sh[kT / 32];
  if (int(blockIdx.x) >= s.n_chunks) {
    const int k = (int(blockIdx.x) - s.n_chunks) * kT + int(threadIdx.x);
    if (k < s.n_orphans) st3(d, s.orphans[k], F3{0.f, 0.f, 0.f});
    return;
  }
  const int begin = s.chunk[3 * blockIdx.x + 1], end = s.chunk[3 * blockIdx.x + 2];
  const int e = begin + int(threadIdx.x);
  double rz = 0.0, rr = 0.0;
  double q[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (e < end) {
    const int v = s.vert[e];
    const F3 r = ld3(b, v), z = apply_block(s.pinv, v, r);
    st3(s.r, v, r); st3(s.z, v, z); st3(d, v, F3{0.f, 0.f, 0.f});
    rz = dot3(r, z); rr = dot3(r, r);
    if constexpr (COARSE) coarse_outer(r, co.Y, e, q);
  }
  rz = block_sum<kT>(rz, sh);
  rr = block_sum<kT>(rr, sh);
  if (threadIdx.x == 0) { s.part[kPartCols * size_t(blockIdx.x) + kRz] = rz; s.part[kPartCols * size_t(blockIdx.x) + kRr] = rr; }
  if constexpr (COARSE) {
    __shared__ double sh9[kT / 32 * 9];
    block_sum9<kT>(q, sh9, co.rpart + 9 * size_t(blockIdx.x));
  }
}

__global__ void __launch_bounds__(kT) pcg_init_kernel(const PcgParams s, const float *__restrict__ b, float *__restrict__ d) {
  pcg_init_body<false>(s, b, d, CoarseParams{});
}

__global__ void __launch_bounds__(kT) pcg_init_coarse_kernel(const PcgParams s, const float *__restrict__ b, float *__restrict__ d,
                                                             const CoarseParams co) {
  pcg_init_body<true>(s, b, d, co);
}

// Hp + mu p with one rounding per entry, in curvature and update alike
__device__ __forceinline__ F3 shifted(F3 hp, F3 p, float mu) {
  return F3{fmaf(mu, p.x, hp.x), fmaf(mu, p.y, hp.y), fmaf(mu, p.z, hp.z)};
}

// Partial of p.Hp (SHIFT: p.(Hp + mu_c p)) of every chunk of an active component.
template <bool SHIFT>
__global__ void __launch_bounds__(kT) pcg_curv_kernel(const PcgParams s, const float *__restrict__ shift) {
  __shared__ double sh[kT / 32];
  const int c = s.chunk[3 * blockIdx.x];
  if (s.comp[c].st_dir != kPcgActive) return;
  const int begin = s.chunk[3 * blockIdx.x + 1], end = s.chunk[3 * blockIdx.x + 2];
  const int e = begin + int(threadIdx.x);
  double q = 0.0;
  if (e < end) {
    const int v = s.vert[e];
    const F3 p = ld3(s.p, v);
    q = dot3(p, SHIFT ? shifted(ld3(s.Hp, v), p, shift[c]) : ld3(s.Hp, v));
  }
  q = block_sum<kT>(q, sh);
  if (threadIdx.x == 0) s.part[kPartCols * size_t(blockIdx.x) + kPHp] = q;
}

// tau >= 0 with |d + tau p|_M = Delta from the recurrences, in the form without cancellation (Delta2 = Delta^2); 0 when
// d is already on or outside the boundary or p has no length
__device__ __forceinline__ double boundary_tau(double pMp, double dMp, double dMd, double Delta2) {
  const double num = Delta2 - dMd;
  const double den = dMp + sqrt(dMp * dMp + pMp * num);
  return num > 0.0 && den > 0.0 ? num / den : 0.0;
}

// alpha = r.z / p.Hp per component; p.Hp <= 0 stops the component (at the first direction d = z = P b), otherwise
// d += alpha p, r -= alpha Hp, z = P r and the partials of the new r.z and r.r.  SHIFT: Hp + mu_c p in place of Hp.
// TR, with a finite radius Delta_c: p.Hp <= 0, or a step that would end at |d + alpha p|_M >= Delta_c, stops the component
// on the boundary instead, d += tau p (NEGCURV_BOUNDARY, BOUNDARY); r and z are then left as they were.  With Delta_c =
// +inf every value written is the one TR = false writes.  COARSE: also the partials of R = Z^T r, and NEGCURV_FIRST takes
// d = p, the first direction (the two-level z).
template <bool SHIFT, bool TR, bool COARSE>
__device__ __forceinline__ void pcg_update_body(const PcgParams &s, float *__restrict__ d, int iter, const float *__restrict__ shift,
                                                const TrParams &t, const CoarseParams &co) {
  __shared__ double sh[kT / 32];
  const int c = s.chunk[3 * blockIdx.x];
  const bool lead = int(blockIdx.x) == s.comp_chunk[c] && threadIdx.x == 0;
  PcgComp &C = s.comp[c];
  const int st = C.st_dir;
  if (st != kPcgActive) {
    if (lead) { C.st_upd = st; C.idle = 1; }
    return;
  }
  const double pHp = fold(s.part, kPHp, s.comp_chunk[c], s.comp_chunk[c + 1], sh);
  const double rz = C.rz;
  const int begin = s.chunk[3 * blockIdx.x + 1], end = s.chunk[3 * blockIdx.x + 2];
  const int e = begin + int(threadIdx.x);
  if (TR) {
    const float rf = t.radius[c];
    const double D = rf > 0.f ? double(rf) : 0.0;     // NaN and <= 0: radius 0
    if (D < INFINITY) {
      const double pMp = t.comp[c].pMp, dMp = t.comp[c].dMp, dMd = t.comp[c].dMd;   // not .step: the lead writes it
      const double D2 = D * D;
      int bst = kPcgActive;                              // stays so for a step inside the radius
      if (!(pHp > 0.0)) {
        bst = TSB_PCG_NEGCURV_BOUNDARY;
      } else {
        const double a = rz / pHp;
        if (dMd + 2.0 * a * dMp + a * a * pMp >= D2) bst = TSB_PCG_BOUNDARY;
      }
      if (bst != kPcgActive) {
        const double tau = boundary_tau(pMp, dMp, dMd, D2);
        const float a = float(tau);
        if (e < end) {
          const int v = s.vert[e];
          const F3 p = ld3(s.p, v);
          F3 x = ld3(d, v);
          x.x += a * p.x; x.y += a * p.y; x.z += a * p.z;
          st3(d, v, x);
        }
        if (lead) { C.st_upd = bst; C.idle = 0; C.n_hvp = iter + 1; C.dHd += tau * tau * pHp; t.comp[c].step = tau; }
        return;
      }
    }
  }
  if (!(pHp > 0.0)) {
    if (iter == 0 && e < end) { const int v = s.vert[e]; st3(d, v, ld3(COARSE ? s.p : s.z, v)); }
    if (lead) { C.st_upd = iter == 0 ? TSB_PCG_NEGCURV_FIRST : TSB_PCG_NEGCURV; C.idle = 0; C.n_hvp = iter + 1; }
    if (TR && lead) t.comp[c].step = iter == 0 ? 1.0 : 0.0;
    return;
  }
  const double alpha = rz / pHp;
  const float a = float(alpha);
  double nrz = 0.0, nrr = 0.0;
  double q[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (e < end) {
    const int v = s.vert[e];
    const F3 p = ld3(s.p, v), hp = SHIFT ? shifted(ld3(s.Hp, v), p, shift[c]) : ld3(s.Hp, v);
    F3 x = ld3(d, v), r = ld3(s.r, v);
    x.x += a * p.x; x.y += a * p.y; x.z += a * p.z;
    r.x -= a * hp.x; r.y -= a * hp.y; r.z -= a * hp.z;
    const F3 z = apply_block(s.pinv, v, r);
    st3(d, v, x); st3(s.r, v, r); st3(s.z, v, z);
    nrz = dot3(r, z); nrr = dot3(r, r);
    if constexpr (COARSE) coarse_outer(r, co.Y, e, q);
  }
  nrz = block_sum<kT>(nrz, sh);
  nrr = block_sum<kT>(nrr, sh);
  if (threadIdx.x == 0) { s.part[kPartCols * size_t(blockIdx.x) + kRz] = nrz; s.part[kPartCols * size_t(blockIdx.x) + kRr] = nrr; }
  if (lead) { C.st_upd = kPcgActive; C.idle = 0; C.n_hvp = iter + 1; C.rz_prev = rz; C.dHd += alpha * alpha * pHp; }
  if (TR && lead) t.comp[c].step = alpha;
  if constexpr (COARSE) {
    __shared__ double sh9[kT / 32 * 9];
    block_sum9<kT>(q, sh9, co.rpart + 9 * size_t(blockIdx.x));
  }
}

template <bool SHIFT, bool TR>
__global__ void __launch_bounds__(kT) pcg_update_kernel(const PcgParams s, float *__restrict__ d, int iter,
                                                        const float *__restrict__ shift, const TrParams t) {
  pcg_update_body<SHIFT, TR, false>(s, d, iter, shift, t, CoarseParams{});
}

template <bool SHIFT, bool TR>
__global__ void __launch_bounds__(kT) pcg_update_coarse_kernel(const PcgParams s, float *__restrict__ d, int iter,
                                                               const float *__restrict__ shift, const TrParams t, const CoarseParams co) {
  pcg_update_body<SHIFT, TR, true>(s, d, iter, shift, t, co);
}

// The trust-region recurrences (TR), advanced by the lead (Steihaug; r^T p_k = 0 and d_k^T M z_{k+1} = r_{k+1}^T d_k = 0):
//   FIRST: pMp = r.z, dMp = dMd = 0;  after a step s along p:  dMd += 2 s dMp + s^2 pMp, and, if still active,
//   dMp = beta (dMp + s pMp), pMp = r.z + beta^2 pMp (beta the fp32 value p is formed with, old pMp on the right).
__device__ __forceinline__ void tr_advance(TrComp &T, bool active, double beta, double rz) {
  const double a = T.step, pMp = T.pMp, dMp = T.dMp;
  T.dMd = T.dMd + 2.0 * a * dMp + a * a * pMp;
  if (active) {
    T.dMp = beta * (dMp + a * pMp);
    T.pMp = rz + beta * beta * pMp;
  }
}

// Folds r.z and r.r, tests convergence and sets the next direction p = z + beta p; a stopped component gets p = 0, so
// later products leave it untouched.  FIRST: the direction of iteration 0 (p = z), which also initialises the state.
// TR: the lead also advances the trust-region recurrences.  COARSE: z is the two-level z + Z E+ R, so r.z gains R^T E+ R
// (R = Z^T r folded from the chunk partials, every chunk for itself) and p gains (Z E+ R)_v.
template <bool FIRST, bool TR, bool COARSE>
__device__ __forceinline__ void pcg_dir_body(const PcgParams s, float rtol, const TrParams t, const CoarseParams co) {
  __shared__ double sh[kT / 32];
  const int c = s.chunk[3 * blockIdx.x];
  const bool lead = int(blockIdx.x) == s.comp_chunk[c] && threadIdx.x == 0;
  PcgComp &C = s.comp[c];
  if (!FIRST && C.idle) return;
  int st = FIRST ? kPcgActive : C.st_upd;
  float beta = 0.f;
  if (st == kPcgActive) {
    const double2 f0 = make_double2(fold(s.part, kRz, s.comp_chunk[c], s.comp_chunk[c + 1], sh),
                                    fold(s.part, kRr, s.comp_chunk[c], s.comp_chunk[c + 1], sh));   // (r.z, r.r)
    const double2 f = COARSE ? make_double2(f0.x + coarse_fold(co, c, s.comp_chunk[c], s.comp_chunk[c + 1], coarse_shared()), f0.y)
                             : f0;
    if (FIRST) {
      if (f.y == 0.0) st = TSB_PCG_ZERO_RHS;
      if (lead) { C.rz = f.x; C.rz_prev = f.x; C.bb = f.y; C.rr = f.y; C.dHd = 0.0; C.st_upd = st; C.idle = 0; C.n_hvp = 0; }
      if (TR && lead) { t.comp[c].pMp = f.x; t.comp[c].dMp = 0.0; t.comp[c].dMd = 0.0; }
    } else {
      if (sqrt(f.y) <= double(rtol) * sqrt(C.bb)) st = TSB_PCG_CONVERGED;
      beta = float(f.x / C.rz_prev);
      if (lead) { C.rz = f.x; C.rr = f.y; if (TR) tr_advance(t.comp[c], st == kPcgActive, double(beta), f.x); }
    }
  } else if (TR && !FIRST && lead) {     // stopped by the update (boundary, negative curvature): its last step still counts
    tr_advance(t.comp[c], false, 0.0, 0.0);
  }
  if (lead) C.st_dir = st;
  const int begin = s.chunk[3 * blockIdx.x + 1], end = s.chunk[3 * blockIdx.x + 2];
  const int e = begin + int(threadIdx.x);
  if (e < end) {
    const int v = s.vert[e];
    F3 p{0.f, 0.f, 0.f};
    if (st == kPcgActive) {
      p = ld3(s.z, v);
      if constexpr (COARSE) { const F3 g = coarse_prolong(coarse_shared() + 9, co.Y, e); p.x += g.x; p.y += g.y; p.z += g.z; }
      if (!FIRST) { const F3 q = ld3(s.p, v); p.x += beta * q.x; p.y += beta * q.y; p.z += beta * q.z; }
    }
    st3(s.p, v, p);
  }
}

template <bool FIRST, bool TR>
__global__ void __launch_bounds__(kT) pcg_dir_kernel(const PcgParams s, float rtol, const TrParams t) {
  pcg_dir_body<FIRST, TR, false>(s, rtol, t, CoarseParams{});
}

template <bool FIRST, bool TR>
__global__ void __launch_bounds__(kT) pcg_dir_coarse_kernel(const PcgParams s, float rtol, const TrParams t, const CoarseParams co) {
  pcg_dir_body<FIRST, TR, true>(s, rtol, t, co);
}

// Components still active, for the host's termination test every check_every iterations.
__global__ void __launch_bounds__(kT) pcg_count_kernel(const PcgParams s) {
  __shared__ int cnt;
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  int k = 0;
  for (int c = int(threadIdx.x); c < s.n_components; c += kT) k += s.comp[c].st_dir == kPcgActive;
  if (k) atomicAdd(&cnt, k);
  __syncthreads();
  if (threadIdx.x == 0) *s.active = cnt;
}

// Partial of b.d of every chunk.
__global__ void __launch_bounds__(kT) pcg_bdotd_kernel(const PcgParams s, const float *__restrict__ b, const float *__restrict__ d) {
  __shared__ double sh[kT / 32];
  const int begin = s.chunk[3 * blockIdx.x + 1], end = s.chunk[3 * blockIdx.x + 2];
  const int e = begin + int(threadIdx.x);
  double q = 0.0;
  if (e < end) { const int v = s.vert[e]; q = dot3(ld3(b, v), ld3(d, v)); }
  q = block_sum<kT>(q, sh);
  if (threadIdx.x == 0) s.part[kPartCols * size_t(blockIdx.x) + kPHp] = q;
}

// One tsb_pcg_sphere_t per component (thread = component).
__global__ void __launch_bounds__(kT) pcg_record_kernel(const PcgParams s, tsb_pcg_sphere_t *__restrict__ out) {
  const int c = blockIdx.x * kT + int(threadIdx.x);
  if (c >= s.n_components) return;
  const PcgComp C = s.comp[c];
  const int k0 = s.comp_chunk[c], k1 = s.comp_chunk[c + 1];
  double bd = 0.0;
  for (int k = k0; k < k1; ++k) bd += s.part[kPartCols * size_t(k) + kPHp];
  tsb_pcg_sphere_t o;
  o.status = C.st_dir == kPcgActive ? TSB_PCG_MAXITER : C.st_dir;
  o.rel_residual = o.status == TSB_PCG_ZERO_RHS ? 0.f : o.status == TSB_PCG_NEGCURV_FIRST ? 1.f : float(sqrt(C.rr / C.bb));
  o.b_dot_d = float(bd);
  o.d_H_d = float(C.dHd);
  o.n_hvp = C.n_hvp;
  o.first_vertex = s.vert[s.chunk[3 * size_t(k0) + 1]];
  o.n_vertices = s.chunk[3 * size_t(k1 - 1) + 2] - s.chunk[3 * size_t(k0) + 1];
  o.reserved = 0;
  out[c] = o;
}

// out = x + a[component] d; CTAs past the chunk table copy the orphan vertices.  out may alias x.
__global__ void __launch_bounds__(kT) sphere_axpy_kernel(const PcgParams s, const float *x, const float *__restrict__ a,
                                                         const float *__restrict__ d, float *out) {
  if (int(blockIdx.x) >= s.n_chunks) {
    const int k = (int(blockIdx.x) - s.n_chunks) * kT + int(threadIdx.x);
    if (k < s.n_orphans) { const int v = s.orphans[k]; st3(out, v, ld3(x, v)); }
    return;
  }
  const int e = s.chunk[3 * blockIdx.x + 1] + int(threadIdx.x);
  if (e >= s.chunk[3 * blockIdx.x + 2]) return;
  const int v = s.vert[e];
  const float al = a[s.chunk[3 * blockIdx.x]];
  const F3 q = ld3(d, v);
  F3 y = ld3(x, v);
  y.x += al * q.x; y.y += al * q.y; y.z += al * q.z;
  st3(out, v, y);
}

// ---- Damped Newton step (tsb_newton_step): the small kernels around the solve and the line search -------------------
// Newton partial table: three columns per chunk, each written by one kernel and folded only by a later one.
constexpr int kNwCols = 3, kNwMaxD = 0, kNwBd = 1, kNwDd = 2;

// Maximum of v over the CTA; valid in thread 0 (a max does not depend on the order).
__device__ __forceinline__ double block_max(double v, double *sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double m = -INFINITY;
  if (threadIdx.x == 0)
#pragma unroll
    for (int w = 0; w < kT / 32; ++w) m = fmax(m, sh[w]);
  return m;
}

// b_c = 0 on the components already frozen; per-chunk maximum of the diagonal entries (D_v)_ii.  PROX: b_c = 0 also where
// w_c is unusable, and elsewhere b_v += (-w_c)(x_v - y_v), each operation rounded on its own (no contraction), as eager
// torch rounds b + (-w) * (x - y); w_c = 0 leaves b as it is.
template <bool PROX>
__global__ void __launch_bounds__(kT) newton_prep_kernel(const PcgParams s, const NewtonParams w, const ProxParams p) {
  __shared__ double sh[kT / 32];
  const int c = s.chunk[3 * blockIdx.x];
  const int e = s.chunk[3 * blockIdx.x + 1] + int(threadIdx.x);
  double m = -INFINITY;
  if (e < s.chunk[3 * blockIdx.x + 2]) {
    const int v = s.vert[e];
    if (PROX) {
      const float wc = p.weight[c];
      if (w.comp[c].status != TSB_NEWTON_ACTIVE || !prox_weight_ok(wc)) {
        st3(w.b, v, F3{0.f, 0.f, 0.f});
      } else if (wc != 0.f) {
        const F3 b = ld3(w.b, v), x = ld3(p.x, v), y = ld3(p.anchor, v);
        st3(w.b, v, F3{__fadd_rn(b.x, __fmul_rn(-wc, __fsub_rn(x.x, y.x))), __fadd_rn(b.y, __fmul_rn(-wc, __fsub_rn(x.y, y.y))),
                       __fadd_rn(b.z, __fmul_rn(-wc, __fsub_rn(x.z, y.z)))});
      }
    } else if (w.comp[c].status != TSB_NEWTON_ACTIVE) {
      st3(w.b, v, F3{0.f, 0.f, 0.f});
    }
    const F3 q = ld3(w.diag, v);
    m = fmax(double(q.x), fmax(double(q.y), double(q.z)));
  }
  m = block_max(m, sh);
  if (threadIdx.x == 0) w.part[kNwCols * size_t(blockIdx.x) + kNwMaxD] = m;
}

// mu_c = tau * max (D_v)_ii on a component's first step (clamped to [mu_min, mu_max]), nu_c = 2; the fp32 shift of the
// solve (thread = component).  PROX: mu_c = tau * (max (D_v)_ii + w_c) and the shift is mu_c + w_c (w_c read as 0 where
// it is unusable: that component's right-hand side is 0).
template <bool PROX>
__global__ void __launch_bounds__(kT) newton_shift_kernel(const PcgParams s, const NewtonParams w, NewtonRule r, const ProxParams p) {
  const int c = blockIdx.x * kT + int(threadIdx.x);
  if (c >= s.n_components) return;
  NewtonComp &N = w.comp[c];
  double wc = 0.0;
  if (PROX) { const float q = p.weight[c]; wc = prox_weight_ok(q) ? double(q) : 0.0; }
  if (!N.init) {
    double m = -INFINITY;
    for (int k = s.comp_chunk[c]; k < s.comp_chunk[c + 1]; ++k) m = fmax(m, w.part[kNwCols * size_t(k) + kNwMaxD]);
    N.mu = fmin(double(r.mu_max), fmax(double(r.mu_min), double(r.tau) * (PROX ? m + wc : m)));
    N.nu = 2.0;
    N.init = 1;
  }
  w.shift[c] = float(PROX ? N.mu + wc : N.mu);
}

// Per-chunk partials of b.d and d.d (b.d exactly as pcg_bdotd_kernel forms it).  PROX: also d.(x - y), in its own array.
template <bool PROX>
__global__ void __launch_bounds__(kT) newton_dots_kernel(const PcgParams s, const NewtonParams w, const ProxParams p) {
  __shared__ double sh[kT / 32];
  const int e = s.chunk[3 * blockIdx.x + 1] + int(threadIdx.x);
  double dd = 0.0, bd = 0.0, dx = 0.0;
  if (e < s.chunk[3 * blockIdx.x + 2]) {
    const int v = s.vert[e];
    const F3 d = ld3(w.d, v);
    bd = dot3(ld3(w.b, v), d);
    dd = dot3(d, d);
    if (PROX) {
      const F3 x = ld3(p.x, v), y = ld3(p.anchor, v);
      dx = double(d.x) * (double(x.x) - double(y.x)) + double(d.y) * (double(x.y) - double(y.y)) +
           double(d.z) * (double(x.z) - double(y.z));
    }
  }
  bd = block_sum<kT>(bd, sh);
  dd = block_sum<kT>(dd, sh);
  if (PROX) dx = block_sum<kT>(dx, sh);
  if (threadIdx.x == 0) {
    w.part[kNwCols * size_t(blockIdx.x) + kNwBd] = bd;
    w.part[kNwCols * size_t(blockIdx.x) + kNwDd] = dd;
    if (PROX) p.part[blockIdx.x] = dx;
  }
}

// The step choice and the damping update of every component (thread = component); see tsb_newton_step and
// tsb_newton_prox_step in the header.
template <bool PROX>
__global__ void __launch_bounds__(kT) newton_decide_kernel(const PcgParams s, const NewtonParams w, NewtonRule r,
                                                           tsb_newton_sphere_t *__restrict__ out, const ProxParams p) {
  const int c = blockIdx.x * kT + int(threadIdx.x);
  if (c >= s.n_components) return;
  const PcgComp C = s.comp[c];
  NewtonComp N = w.comp[c];
  const int k0 = s.comp_chunk[c], k1 = s.comp_chunk[c + 1];
  double bd = 0.0, dd = 0.0, dx = 0.0;
  for (int k = k0; k < k1; ++k) bd += w.part[kNwCols * size_t(k) + kNwBd];
  for (int k = k0; k < k1; ++k) dd += w.part[kNwCols * size_t(k) + kNwDd];
  double wc = 0.0;
  bool bad_w = false;
  if (PROX) {
    for (int k = k0; k < k1; ++k) dx += p.part[k];
    const float q = p.weight[c];
    bad_w = !prox_weight_ok(q);
    wc = bad_w ? 0.0 : double(q);
  }
  const double bdf = double(float(bd)), dHd = double(float(C.dHd));   // the values the solve's records report
  const double g = sqrt(C.bb);
  int ks = -1;
  float alpha = 0.f, delta = 0.f;
  double rho = 0.0;
  if (N.status == TSB_NEWTON_ACTIVE) {
    if (PROX && bad_w) {
      N.status = TSB_NEWTON_STALLED;
    } else if (g <= double(r.gtol)) {
      N.status = TSB_NEWTON_CONVERGED;
    } else {
      const float *dl = w.sphere_delta + size_t(c) * size_t(r.n_alpha) * 4;
      const double lim = double(r.eta) * double(w.sphere_step[c]);
      if (bdf > 0.0)
        for (int k = 0; k < r.n_alpha; ++k) {
          const double a = double(w.alphas[k]);
          if (a < lim && step_change<PROX>(dl[4 * k], wc, a, dx, dd) <= -double(r.sigma) * a * bdf) { ks = k; break; }
        }
      const double pred = bdf - 0.5 * (dHd - (PROX ? double(w.shift[c]) - wc : double(w.shift[c])) * dd);
      rho = pred > 0.0 ? -step_change<PROX>(dl[0], wc, double(w.alphas[0]), dx, dd) / pred : 1.0;
      if (ks == 0) {
        const double t = 2.0 * rho - 1.0;
        N.mu = fmax(double(r.mu_min), N.mu * fmax(1.0 / 3.0, 1.0 - t * t * t));
        N.nu = 2.0;
      } else {
        N.mu = fmin(double(r.mu_max), N.mu * N.nu);
        N.nu *= 2.0;
      }
      if (ks < 0 && N.mu == double(r.mu_max)) N.status = TSB_NEWTON_STALLED;
      if (ks >= 0) {
        alpha = w.alphas[ks];
        delta = PROX ? float(step_change<PROX>(dl[4 * ks], wc, double(alpha), dx, dd)) : dl[4 * ks];
      }
    }
  }
  w.alpha_sphere[c] = alpha;
  w.comp[c] = N;
  if (!out) return;
  tsb_newton_sphere_t o;
  o.mu = N.mu;
  o.rho = rho;
  o.grad_norm = float(g);
  o.alpha = alpha;
  o.delta = delta;
  o.b_dot_d = float(bd);
  o.k = ks;
  o.pcg_status = C.st_dir == kPcgActive ? TSB_PCG_MAXITER : C.st_dir;
  o.n_hvp = C.n_hvp;
  o.status = N.status;
  o.first_vertex = s.vert[s.chunk[3 * size_t(k0) + 1]];
  o.reserved[0] = o.reserved[1] = o.reserved[2] = 0;
  out[c] = o;
}

// ---- Trust-region Newton step (tsb_newton_tr_step) -------------------------------------------------------------------
// It reuses the prep kernels above (their max (D_v)_ii column is not read in this step) and puts the per-chunk partials
// of b^T P b in that column instead: written by newton_tr_bpb_kernel, folded by newton_tr_radius_kernel.

// Partial of b^T P b of every chunk of a component whose radius is not yet initialised (P: the blocks just set).
__global__ void __launch_bounds__(kT) newton_tr_bpb_kernel(const PcgParams s, const NewtonParams w, const NewtonTrParams t) {
  __shared__ double sh[kT / 32];
  if (t.state[s.chunk[3 * blockIdx.x]].init) return;
  const int e = s.chunk[3 * blockIdx.x + 1] + int(threadIdx.x);
  double q = 0.0;
  if (e < s.chunk[3 * blockIdx.x + 2]) {
    const int v = s.vert[e];
    const F3 b = ld3(w.b, v);
    q = dot3(b, apply_block(s.pinv, v, b));
  }
  q = block_sum<kT>(q, sh);
  if (threadIdx.x == 0) w.part[kNwCols * size_t(blockIdx.x) + kNwMaxD] = q;
}

// Delta_c = clamp(radius_init sqrt(b^T P b), radius_min, radius_max) on a component's first step after a reset, and the
// fp32 radius of the solve (thread = component).
__global__ void __launch_bounds__(kT) newton_tr_radius_kernel(const PcgParams s, const NewtonParams w, const NewtonTrParams t,
                                                              const NewtonTrRule r) {
  const int c = blockIdx.x * kT + int(threadIdx.x);
  if (c >= s.n_components) return;
  TrState S = t.state[c];
  if (!S.init) {
    double bpb = 0.0;
    for (int k = s.comp_chunk[c]; k < s.comp_chunk[c + 1]; ++k) bpb += w.part[kNwCols * size_t(k) + kNwMaxD];
    S.radius = fmin(double(r.radius_max), fmax(double(r.radius_min), double(r.radius_init) * sqrt(bpb)));
    S.init = 1;
    t.state[c] = S;
  }
  t.radius[c] = float(S.radius);
}

// Acceptance and radius update of every component (thread = component); see tsb_newton_tr_step in the header.  LS: a
// step the trust-region rule rejects is backtracked to the largest 2^-k (k >= 1) of the line search with the Armijo
// decrease below the inversion bound (tsb_newton_tr_step_ex); the backtracking options b are read only then.
template <bool PROX, bool LS>
__global__ void __launch_bounds__(kT) newton_decide_tr_kernel(const PcgParams s, const NewtonParams w, const NewtonTrParams t,
                                                              const NewtonTrRule r, tsb_newton_tr_sphere_t *__restrict__ out,
                                                              const ProxParams p, const NewtonBacktrack b) {
  const int c = blockIdx.x * kT + int(threadIdx.x);
  if (c >= s.n_components) return;
  const PcgComp C = s.comp[c];
  NewtonComp N = w.comp[c];
  TrState S = t.state[c];
  const double dMd = t.tr[c].dMd;
  const int k0 = s.comp_chunk[c], k1 = s.comp_chunk[c + 1];
  double bd = 0.0, dd = 0.0, dx = 0.0;
  for (int k = k0; k < k1; ++k) bd += w.part[kNwCols * size_t(k) + kNwBd];
  for (int k = k0; k < k1; ++k) dd += w.part[kNwCols * size_t(k) + kNwDd];
  double wc = 0.0;
  bool bad_w = false;
  if (PROX) {
    for (int k = k0; k < k1; ++k) dx += p.part[k];
    const float q = p.weight[c];
    bad_w = !prox_weight_ok(q);
    wc = bad_w ? 0.0 : double(q);
  }
  const double bdf = double(float(bd)), dHd = double(float(C.dHd));   // the values the solve's records report
  const double g = sqrt(C.bb), dn = sqrt(dMd);
  const int pst = C.st_dir == kPcgActive ? TSB_PCG_MAXITER : C.st_dir;
  float alpha = 0.f, delta = 0.f;
  double rho = 0.0, pred = 0.0;
  if (N.status == TSB_NEWTON_ACTIVE) {
    if (PROX && bad_w) {
      N.status = TSB_NEWTON_STALLED;
    } else if (g <= double(r.gtol)) {
      N.status = TSB_NEWTON_CONVERGED;
    } else {
      pred = bdf - 0.5 * dHd;
      const float *dl = w.sphere_delta + (LS ? size_t(c) * size_t(b.n_alpha) * 4 : 4 * size_t(c));   // [n_alpha][4]
      const double dphi = step_change<PROX>(dl[0], wc, 1.0, dx, dd);
      if (pred > 0.0) rho = -dphi / pred;
      const double lim = double(r.eta) * double(w.sphere_step[c]);
      const bool flips = !(1.0 < lim);
      const double r0 = S.radius;
      if (flips) S.radius = fmin(0.25 * S.radius, lim * dn);
      else if (!(rho >= 0.25)) S.radius = 0.25 * dn;
      else if (rho > 0.75 && (pst == TSB_PCG_BOUNDARY || pst == TSB_PCG_NEGCURV_BOUNDARY))
        S.radius = fmin(2.0 * S.radius, double(r.radius_max));
      int ks = -1;
      if (!flips && pred > 0.0 && rho > double(r.accept)) {
        alpha = 1.f;
        delta = float(dphi);
      } else {
        if (LS && bdf > 0.0)
          for (int k = 1; k < b.n_alpha; ++k) {
            const double a = double(w.alphas[k]);
            if (a < lim && step_change<PROX>(dl[4 * k], wc, a, dx, dd) <= -double(b.sigma) * a * bdf) { ks = k; break; }
          }
        if (LS && ks > 0) {       // the radius shrinks by at most the quarter of a poor model, to no less than the step
          alpha = w.alphas[ks];
          delta = float(step_change<PROX>(dl[4 * ks], wc, double(alpha), dx, dd));
          S.radius = fmin(double(r.radius_max), fmax(double(r.radius_min), fmax(double(alpha) * dn, 0.25 * r0)));
        } else if (S.radius < double(r.radius_min)) {
          N.status = TSB_NEWTON_STALLED;
        }
      }
    }
  }
  w.alpha_sphere[c] = alpha;
  w.comp[c] = N;
  t.state[c] = S;
  if (!out) return;
  tsb_newton_tr_sphere_t o;
  o.radius = S.radius;
  o.rho = rho;
  o.grad_norm = float(g);
  o.alpha = alpha;
  o.delta = delta;
  o.b_dot_d = float(bd);
  o.pred = float(pred);
  o.d_norm = float(dn);
  o.pcg_status = pst;
  o.n_hvp = C.n_hvp;
  o.status = N.status;
  o.first_vertex = s.vert[s.chunk[3 * size_t(k0) + 1]];
  o.reserved[0] = o.reserved[1] = 0;
  out[c] = o;
}

unsigned with_orphans(const PcgParams &s) { return unsigned(s.n_chunks + (s.n_orphans + kT - 1) / kT); }
unsigned comp_blocks(const PcgParams &s) { return unsigned((s.n_components + kT - 1) / kT); }   // thread = component

}  // namespace

cudaError_t launch_pcg_blocks(const PcgParams &s, const float *diag, float rel_floor, float *inv_out, cudaStream_t st) {
  pcg_blocks_kernel<<<unsigned((s.n + kT - 1) / kT), kT, 0, st>>>(diag, s.n, rel_floor, s.pinv, inv_out);
  return cudaGetLastError();
}

cudaError_t launch_pcg_blocks_shift(const PcgParams &s, const float *diag, float rel_floor, const float *shift, float *inv_out,
                                    cudaStream_t st) {
  pcg_blocks_shift_kernel<<<with_orphans(s), kT, 0, st>>>(s, diag, rel_floor, shift, inv_out);
  return cudaGetLastError();
}

// The symmetric Gauss-Seidel mode runs the init and update kernels as they are and overwrites the z and the r.z / r.r
// partials they wrote (block Jacobi's) with the sweep's, before the direction kernel folds them.
// The coarse space adds its term in the direction kernel, after the sweep: the init and update kernels' R partials are
// of r, which the sweep does not change.
cudaError_t launch_pcg_begin(const PcgParams &s, const float *b, float *d, const TrParams *tr, cudaStream_t st,
                             const SgsParams *sgs, const CoarseParams *co) {
  if (co) pcg_init_coarse_kernel<<<with_orphans(s), kT, 0, st>>>(s, b, d, *co);
  else pcg_init_kernel<<<with_orphans(s), kT, 0, st>>>(s, b, d);
  if (sgs) {
    const cudaError_t e = launch_sgs_sweep(s, *sgs, SgsSweep{b, s.z, s.part, kPartCols, kRz, kRr, nullptr, nullptr}, st);
    if (e != cudaSuccess) return e;
  }
  const TrParams t = tr ? *tr : TrParams{};
  if (co) (tr ? pcg_dir_coarse_kernel<true, true> : pcg_dir_coarse_kernel<true, false>)<<<unsigned(s.n_chunks), kT, 0, st>>>(s, 0.f, t, *co);
  else (tr ? pcg_dir_kernel<true, true> : pcg_dir_kernel<true, false>)<<<unsigned(s.n_chunks), kT, 0, st>>>(s, 0.f, t);
  return cudaGetLastError();
}

cudaError_t launch_pcg_step(const PcgParams &s, float *d, int iter, float rtol, const float *shift, const TrParams *tr,
                            cudaStream_t st, const SgsParams *sgs, const CoarseParams *co) {
  const TrParams t = tr ? *tr : TrParams{};
  const unsigned g = unsigned(s.n_chunks);
  (shift ? pcg_curv_kernel<true> : pcg_curv_kernel<false>)<<<g, kT, 0, st>>>(s, shift);
  if (co)
    (shift ? (tr ? pcg_update_coarse_kernel<true, true> : pcg_update_coarse_kernel<true, false>)
           : (tr ? pcg_update_coarse_kernel<false, true> : pcg_update_coarse_kernel<false, false>))<<<g, kT, 0, st>>>(
        s, d, iter, shift, t, *co);
  else
    (shift ? (tr ? pcg_update_kernel<true, true> : pcg_update_kernel<true, false>)
           : (tr ? pcg_update_kernel<false, true> : pcg_update_kernel<false, false>))<<<g, kT, 0, st>>>(s, d, iter, shift, t);
  if (sgs) {
    const cudaError_t e = launch_sgs_sweep(s, *sgs, SgsSweep{s.r, s.z, s.part, kPartCols, kRz, kRr, s.comp, nullptr}, st);
    if (e != cudaSuccess) return e;
  }
  if (co) (tr ? pcg_dir_coarse_kernel<false, true> : pcg_dir_coarse_kernel<false, false>)<<<g, kT, 0, st>>>(s, rtol, t, *co);
  else (tr ? pcg_dir_kernel<false, true> : pcg_dir_kernel<false, false>)<<<g, kT, 0, st>>>(s, rtol, t);
  return cudaGetLastError();
}

cudaError_t launch_pcg_count(const PcgParams &s, cudaStream_t st) {
  pcg_count_kernel<<<1, kT, 0, st>>>(s);
  return cudaGetLastError();
}

cudaError_t launch_pcg_records(const PcgParams &s, const float *b, const float *d, tsb_pcg_sphere_t *out, cudaStream_t st) {
  pcg_bdotd_kernel<<<unsigned(s.n_chunks), kT, 0, st>>>(s, b, d);
  pcg_record_kernel<<<comp_blocks(s), kT, 0, st>>>(s, out);
  return cudaGetLastError();
}

cudaError_t launch_sphere_axpy(const PcgParams &s, const float *x, const float *a, const float *d, float *out, cudaStream_t st) {
  sphere_axpy_kernel<<<with_orphans(s), kT, 0, st>>>(s, x, a, d, out);
  return cudaGetLastError();
}

cudaError_t launch_newton_prep(const PcgParams &s, const NewtonParams &w, const ProxParams *p, cudaStream_t st) {
  (p ? newton_prep_kernel<true> : newton_prep_kernel<false>)<<<unsigned(s.n_chunks), kT, 0, st>>>(s, w, p ? *p : ProxParams{});
  return cudaGetLastError();
}

cudaError_t launch_newton_shift(const PcgParams &s, const NewtonParams &w, const NewtonRule &r, const ProxParams *p,
                                cudaStream_t st) {
  (p ? newton_shift_kernel<true> : newton_shift_kernel<false>)<<<comp_blocks(s), kT, 0, st>>>(s, w, r, p ? *p : ProxParams{});
  return cudaGetLastError();
}

cudaError_t launch_newton_dots(const PcgParams &s, const NewtonParams &w, const ProxParams *p, cudaStream_t st) {
  (p ? newton_dots_kernel<true> : newton_dots_kernel<false>)<<<unsigned(s.n_chunks), kT, 0, st>>>(s, w, p ? *p : ProxParams{});
  return cudaGetLastError();
}

cudaError_t launch_newton_decide(const PcgParams &s, const NewtonParams &w, const NewtonRule &r, const ProxParams *p,
                                 tsb_newton_sphere_t *out, cudaStream_t st) {
  (p ? newton_decide_kernel<true> : newton_decide_kernel<false>)<<<comp_blocks(s), kT, 0, st>>>(s, w, r, out,
                                                                                                 p ? *p : ProxParams{});
  return cudaGetLastError();
}

cudaError_t launch_newton_tr_radius(const PcgParams &s, const NewtonParams &w, const NewtonTrParams &t, const NewtonTrRule &r,
                                    cudaStream_t st, const SgsParams *sgs) {
  if (sgs) {            // z is scratch here: the solve's init overwrites it
    const cudaError_t e = launch_sgs_sweep(s, *sgs, SgsSweep{w.b, s.z, w.part, kNwCols, kNwMaxD, -1, nullptr, t.state}, st);
    if (e != cudaSuccess) return e;
  } else {
    newton_tr_bpb_kernel<<<unsigned(s.n_chunks), kT, 0, st>>>(s, w, t);
  }
  newton_tr_radius_kernel<<<comp_blocks(s), kT, 0, st>>>(s, w, t, r);
  return cudaGetLastError();
}

cudaError_t launch_newton_tr_decide(const PcgParams &s, const NewtonParams &w, const NewtonTrParams &t, const NewtonTrRule &r,
                                    const ProxParams *p, const NewtonBacktrack *bt, tsb_newton_tr_sphere_t *out, cudaStream_t st) {
  (p ? (bt ? newton_decide_tr_kernel<true, true> : newton_decide_tr_kernel<true, false>)
     : (bt ? newton_decide_tr_kernel<false, true> : newton_decide_tr_kernel<false, false>))<<<comp_blocks(s), kT, 0, st>>>(
      s, w, t, r, out, p ? *p : ProxParams{}, bt ? *bt : NewtonBacktrack{});
  return cudaGetLastError();
}

}  // namespace tsb
