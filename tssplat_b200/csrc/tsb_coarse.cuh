// Device helpers of the affine coarse space (CoarseParams in tsb_solver.cuh), shared by the CG kernels (tsb_solver.cu)
// and the coarse kernels (tsb_coarse.cu).  Every sum runs in a fixed order: no atomics.
#pragma once
#include "tsb_device.cuh"
#include "tsb_solver.cuh"

namespace tsb {

// r_e Y_e^T of one solver entry, entry 3 a + b = r[a] Y[b]
__device__ __forceinline__ void coarse_outer(F3 r, const float *__restrict__ Y, int e, double (&q)[9]) {
  const double y0 = Y[3 * size_t(e)], y1 = Y[3 * size_t(e) + 1], y2 = Y[3 * size_t(e) + 2];
  const double ra[3] = {r.x, r.y, r.z};
#pragma unroll
  for (int a = 0; a < 3; ++a) { q[3 * a] = ra[a] * y0; q[3 * a + 1] = ra[a] * y1; q[3 * a + 2] = ra[a] * y2; }
}

// Sum over the CTA of the 9 values q (a shuffle tree per warp, the warps in order); threads 0..8 write out[0..8].
// sh: [NT / 32 * 9] doubles of shared memory no other code of the kernel uses.
template <int NT>
__device__ __forceinline__ void block_sum9(double (&q)[9], double *sh, double *out) {
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    double v = q[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    if ((threadIdx.x & 31) == 0) sh[9 * (threadIdx.x >> 5) + k] = v;
  }
  __syncthreads();
  if (threadIdx.x < 9) {
    double a = 0.0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) a += sh[9 * w + threadIdx.x];
    out[threadIdx.x] = a;
  }
}

// The coarse kernels' 18 doubles of shared memory (R, then G = E+ R), allocated only in the kernels that call this
__device__ __forceinline__ double *coarse_shared() {
  __shared__ double sh[18];
  return sh;
}

// Folds the R partials of chunks [c0, c1) of component c in a fixed order (lane l of warp 0 adds chunks c0 + l,
// c0 + l + 32, ..., a shuffle tree combines the lanes), then G = E+_c R into sh[9..17]; returns R^T G, the same in every
// thread.  sh: [18] doubles of shared memory; G stays there for coarse_prolong.
__device__ __forceinline__ double coarse_fold(const CoarseParams &co, int c, int c0, int c1, double *sh) {
  if (threadIdx.x < 32) {
    double a[9];
#pragma unroll
    for (int j = 0; j < 9; ++j) a[j] = 0.0;
    for (int k = c0 + int(threadIdx.x); k < c1; k += 32)
#pragma unroll
      for (int j = 0; j < 9; ++j) a[j] += co.rpart[9 * size_t(k) + j];
#pragma unroll
    for (int j = 0; j < 9; ++j) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a[j] += __shfl_xor_sync(0xFFFFFFFFu, a[j], o);
      if (threadIdx.x == 0) sh[j] = a[j];
    }
  }
  __syncthreads();
  if (threadIdx.x < 9) {
    const double *E = co.Einv + 81 * size_t(c) + 9 * threadIdx.x;
    double g = 0.0;
#pragma unroll
    for (int j = 0; j < 9; ++j) g += E[j] * sh[j];
    sh[9 + threadIdx.x] = g;
  }
  __syncthreads();
  double rg = 0.0;
#pragma unroll
  for (int j = 0; j < 9; ++j) rg += sh[j] * sh[9 + j];
  return rg;
}

// (Z G)_e = G Y_e, G the 3 x 3 of coarse_fold
__device__ __forceinline__ F3 coarse_prolong(const double *G, const float *__restrict__ Y, int e) {
  const double y0 = Y[3 * size_t(e)], y1 = Y[3 * size_t(e) + 1], y2 = Y[3 * size_t(e) + 2];
  return F3{float(G[0] * y0 + G[1] * y1 + G[2] * y2), float(G[3] * y0 + G[4] * y1 + G[5] * y2),
            float(G[6] * y0 + G[7] * y1 + G[8] * y2)};
}

}  // namespace tsb
