// Multicolour block symmetric Gauss-Seidel preconditioner of the per-component solve (tsb_pcg_enable_sgs in
// include/tssplat_b200.h; DESIGN.md section 5, "Symmetric Gauss-Seidel preconditioner").
//
// One CTA per component.  The component's vector lives in shared memory, 12 bytes per vertex at its position in the
// solver's vertex list.  The forward sweep runs colour by colour, the backward sweep colours in reverse, with a barrier
// between colours; inside a colour no two rows couple, so its rows are independent: a warp takes one row at a time, its
// lanes the row's blocks (32 at a time), and a fixed shuffle tree sums the lanes.  Then z goes to global memory and, chunk
// by chunk in the solver's chunk order, the fp64 partials of r.z and r.r go to the partial table, summed in a fixed
// order (one thread per entry of the chunk, a shuffle tree per warp, the warps in order), so the direction kernel folds
// them as it folds block Jacobi's.  No atomics, and no launch reads what
// another CTA of it writes: bitwise repeatable, and a component's z depends on its own r only.
#include "tsb_device.cuh"
#include "tsb_sgs.cuh"

namespace tsb {
namespace {

constexpr int kT = kSgsT, kW = kT / 32;

// sum over the list [b0, b1) of A_ij v_j (v in shared memory), lanes over the entries, summed by a fixed shuffle tree;
// valid in every lane
__device__ __forceinline__ F3 row_sum(const int2 *__restrict__ list, int b0, int b1, const float *__restrict__ values,
                                      const float *v, int lane) {
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int b = b0 + lane; b < b1; b += 32) {
    const int2 q = list[b];
    const float *A = values + 9 * size_t(q.x);
    const float u0 = v[3 * q.y], u1 = v[3 * q.y + 1], u2 = v[3 * q.y + 2];
    a0 = fmaf(A[0], u0, fmaf(A[1], u1, fmaf(A[2], u2, a0)));
    a1 = fmaf(A[3], u0, fmaf(A[4], u1, fmaf(A[5], u2, a1)));
    a2 = fmaf(A[6], u0, fmaf(A[7], u1, fmaf(A[8], u2, a2)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a0 += __shfl_xor_sync(0xFFFFFFFFu, a0, o);
    a1 += __shfl_xor_sync(0xFFFFFFFFu, a1, o);
    a2 += __shfl_xor_sync(0xFFFFFFFFu, a2, o);
  }
  return F3{a0, a1, a2};
}

__global__ void __launch_bounds__(kT) pcg_sgs_kernel(const PcgParams s, const SgsParams g, const SgsSweep w) {
  extern __shared__ float vec[];          // [3 * vertices of the component]
  __shared__ double sh[kW];
  const int c = int(blockIdx.x);
  if (w.comp && w.comp[c].st_upd != kPcgActive) return;
  if (w.tr_state && w.tr_state[c].init) return;
  const int e0 = g.comp_off[c], nv = g.comp_off[c + 1] - e0;
  const int k0 = g.color_ptr[c], nc = g.color_ptr[c + 1] - k0 - 1;
  const int warp = int(threadIdx.x >> 5), lane = int(threadIdx.x & 31);
  // forward: y_i = Dt_i^-1 (r_i - sum_{earlier colours} A_ij y_j)
  for (int k = 0; k < nc; ++k) {
    for (int q = g.color_off[k0 + k] + warp; q < g.color_off[k0 + k + 1]; q += kW) {
      const int e = g.sched[q], v = s.vert[e];
      const F3 r = ld3(w.r, v);                // issued before the row's sum, which does not depend on it
      const F3 a = row_sum(g.lo, g.lo_ptr[e], g.lo_ptr[e + 1], g.values, vec, lane);
      if (lane == 0) {
        const F3 y = apply_block(s.pinv, v, F3{r.x - a.x, r.y - a.y, r.z - a.z});
        float *o = vec + 3 * (e - e0);
        o[0] = y.x; o[1] = y.y; o[2] = y.z;
      }
    }
    __syncthreads();
  }
  // backward, in place: z_i = y_i - Dt_i^-1 sum_{later colours} A_ij z_j
  for (int k = nc - 2; k >= 0; --k) {     // the last colour has no later blocks: z = y there
    for (int q = g.color_off[k0 + k] + warp; q < g.color_off[k0 + k + 1]; q += kW) {
      const int e = g.sched[q];
      const F3 a = row_sum(g.hi, g.hi_ptr[e], g.hi_ptr[e + 1], g.values, vec, lane);
      if (lane == 0) {
        const F3 t = apply_block(s.pinv, s.vert[e], a);
        float *o = vec + 3 * (e - e0);
        o[0] -= t.x; o[1] -= t.y; o[2] -= t.z;
      }
    }
    __syncthreads();
  }
  // z out, and the partials of every chunk of the component (thread = entry of the chunk, as in the solver; the threads
  // past the chunk size add exact zeros)
  for (int q = int(threadIdx.x); q < nv; q += kT) st3(w.z, s.vert[e0 + q], F3{vec[3 * q], vec[3 * q + 1], vec[3 * q + 2]});
  if (!w.part) return;
  for (int ch = s.comp_chunk[c]; ch < s.comp_chunk[c + 1]; ++ch) {
    const int e = s.chunk[3 * ch + 1] + int(threadIdx.x);
    double rz = 0.0, rr = 0.0;
    if (int(threadIdx.x) < kPcgChunkVerts && e < s.chunk[3 * ch + 2]) {
      const F3 r = ld3(w.r, s.vert[e]);
      const F3 z{vec[3 * (e - e0)], vec[3 * (e - e0) + 1], vec[3 * (e - e0) + 2]};
      rz = dot3(r, z);
      rr = dot3(r, r);
    }
    rz = block_sum<kT>(rz, sh);
    if (w.col_rr >= 0) rr = block_sum<kT>(rr, sh);
    if (threadIdx.x == 0) {
      w.part[size_t(w.stride) * size_t(ch) + w.col_rz] = rz;
      if (w.col_rr >= 0) w.part[size_t(w.stride) * size_t(ch) + w.col_rr] = rr;
    }
  }
}

// The two diagonal planes of the assembled matrix (thread = vertex): (xx, yy, zz) and (yz, xz, xy).
__global__ void __launch_bounds__(256) sgs_diag_kernel(const SgsParams g, int n, float *__restrict__ diag) {
  const int v = int(blockIdx.x) * 256 + int(threadIdx.x);
  if (v >= n) return;
  float d[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int b = g.crow[v]; b < g.crow[v + 1]; ++b)
    if (g.col[b] == v) {
      const float *A = g.values + 9 * size_t(b);
      d[0] = A[0]; d[1] = A[4]; d[2] = A[8]; d[3] = A[5]; d[4] = A[2]; d[5] = A[1];
      break;
    }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    diag[3 * size_t(v) + k] = d[k];
    diag[3 * (size_t(n) + size_t(v)) + k] = d[3 + k];
  }
}

}  // namespace

cudaError_t sgs_configure(int max_comp_verts, int *max_verts) {
  int dev = 0, optin = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  cudaFuncAttributes fa{};
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, pcg_sgs_kernel);
  if (e != cudaSuccess) return e;
  *max_verts = int((size_t(optin) - fa.sharedSizeBytes) / 12);
  if (max_comp_verts > *max_verts || 12 * max_comp_verts <= fa.maxDynamicSharedSizeBytes) return cudaSuccess;
  return cudaFuncSetAttribute(pcg_sgs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 12 * max_comp_verts);
}

cudaError_t launch_sgs_sweep(const PcgParams &s, const SgsParams &g, const SgsSweep &w, cudaStream_t st) {
  if (s.n_components == 0) return cudaSuccess;
  pcg_sgs_kernel<<<unsigned(s.n_components), kT, 12 * size_t(g.max_verts), st>>>(s, g, w);
  return cudaGetLastError();
}

cudaError_t launch_sgs_diag(const SgsParams &g, int n, float *diag_out, cudaStream_t st) {
  sgs_diag_kernel<<<unsigned((n + 255) / 256), 256, 0, st>>>(g, n, diag_out);
  return cudaGetLastError();
}

}  // namespace tsb
