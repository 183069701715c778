// Small device helpers shared by the solver (tsb_solver.cu), the Gauss-Seidel sweep (tsb_sgs.cu), the projected
// Hessian (tsb_psd.cu) and the L-BFGS step (tsb_lbfgs.cu): the fixed-order CTA sum, the per-vertex 3-vector access and
// the proximal step's weight test and objective change.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

namespace tsb {

// Sum of v over an NT-thread CTA in a fixed order (shuffle tree, then the warps in order); valid in thread 0.
template <int NT>
__device__ __forceinline__ double block_sum(double v, double *sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  __syncthreads();                                  // sh may still be read from the previous sum
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) s += sh[w];
  return s;
}

struct F3 { float x, y, z; };
__device__ __forceinline__ F3 ld3(const float *a, int v) { return F3{a[3 * size_t(v)], a[3 * size_t(v) + 1], a[3 * size_t(v) + 2]}; }
__device__ __forceinline__ void st3(float *a, int v, F3 q) { a[3 * size_t(v)] = q.x; a[3 * size_t(v) + 1] = q.y; a[3 * size_t(v) + 2] = q.z; }
__device__ __forceinline__ double dot3(F3 a, F3 b) { return double(a.x) * double(b.x) + double(a.y) * double(b.y) + double(a.z) * double(b.z); }
// z = P r with the symmetric block stored as xx yy zz yz xz xy
__device__ __forceinline__ F3 apply_block(const float *pinv, int v, F3 r) {
  const float *q = pinv + 6 * size_t(v);
  const float xx = q[0], yy = q[1], zz = q[2], yz = q[3], xz = q[4], xy = q[5];
  return F3{xx * r.x + xy * r.y + xz * r.z, xy * r.x + yy * r.y + yz * r.z, xz * r.x + yz * r.y + zz * r.z};
}

// The proximal weight of a component is usable when it is finite and >= 0 (NaN fails both tests).
__device__ __forceinline__ bool prox_weight_ok(float wc) { return wc >= 0.f && wc < INFINITY; }

// Phi_c(x + a d) - Phi_c(x) from the line search's dE = E_c(x + a d) - E_c(x): dE + w_c (a d.(x - y) + a^2 |d|^2 / 2).
// Without PROX, or with w_c = 0, it is dE itself.
template <bool PROX>
__device__ __forceinline__ double step_change(float dE, double wc, double a, double dx, double dd) {
  return PROX && wc > 0.0 ? double(dE) + wc * (a * dx + 0.5 * a * a * dd) : double(dE);
}

}  // namespace tsb
