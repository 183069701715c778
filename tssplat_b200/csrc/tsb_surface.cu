// Surface gather + vertex-normal splat (SURVEY.md section 8(f) rank 2) behind the C ABI.
//
// Replaces, per geometry forward, `self.v_pos = tet_v[surface_vid]` (geometry/tetmesh_geometry.py:33) and
// `_compute_vertex_normal` (geometry/tetmesh_geometry.py:39-66: face normals cross(v1-v0, v2-v0), three
// scatter_add_ splats, the 1e-20 degenerate fallback to (0,0,1), F.normalize) and their autograd backward.
// Same gather-not-scatter idea as the energy kernel: a vertex-to-incident-face CSR built once lets every
// surface vertex SUM its faces in a fixed order -- no atomics, bitwise repeatable (the reference's
// scatter_add_ is not).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/tssplat_b200.h"

struct tsb_surface_s {
  int device = 0;
  int32_t nsv = 0, nsf = 0, n = 0;
  int32_t *svid = nullptr;      // [nsv] tet-mesh vertex of each surface vertex
  int32_t *faces = nullptr;     // [3*nsf] surface-vertex ids
  int32_t *inc_ptr = nullptr;   // [nsv+1]
  int32_t *inc = nullptr;       // [3*nsf] face*4 + corner, ascending per vertex
  float *h = nullptr;           // [3*nsv] backward scratch: gradient w.r.t. the un-normalised normals
  std::string err;
};

namespace {

thread_local std::string g_surface_err;

struct Guard {
  int prev = -1;
  explicit Guard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); }
  ~Guard() { if (prev >= 0) cudaSetDevice(prev); }
};

__device__ __forceinline__ float3 ld3(const float *p, int i) { return make_float3(p[3 * size_t(i)], p[3 * size_t(i) + 1], p[3 * size_t(i) + 2]); }
__device__ __forceinline__ float3 sub3(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 add3(float3 a, float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 cross3(float3 a, float3 b) { return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// un-normalised vertex normal: sum over incident faces of cross(v1 - v0, v2 - v0)   (tetmesh_geometry.py:40-54)
__device__ __forceinline__ float3 raw_normal(int a, const float *tet_v, const int32_t *svid, const int32_t *faces,
                                             const int32_t *inc_ptr, const int32_t *inc) {
  float3 n = make_float3(0.f, 0.f, 0.f);
  for (int e = inc_ptr[a]; e < inc_ptr[a + 1]; ++e) {
    const int f = inc[e] >> 2;
    const float3 v0 = ld3(tet_v, svid[faces[3 * f]]), v1 = ld3(tet_v, svid[faces[3 * f + 1]]), v2 = ld3(tet_v, svid[faces[3 * f + 2]]);
    n = add3(n, cross3(sub3(v1, v0), sub3(v2, v0)));
  }
  return n;
}

__global__ void surface_forward_kernel(const float *__restrict__ tet_v, const int32_t *__restrict__ svid, const int32_t *__restrict__ faces,
                                       const int32_t *__restrict__ inc_ptr, const int32_t *__restrict__ inc, int nsv,
                                       float *__restrict__ v_pos, float *__restrict__ v_nrm) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= nsv) return;
  const float3 p = ld3(tet_v, svid[a]);
  if (v_pos) { v_pos[3 * size_t(a)] = p.x; v_pos[3 * size_t(a) + 1] = p.y; v_pos[3 * size_t(a) + 2] = p.z; }
  if (v_nrm) {
    float3 n = raw_normal(a, tet_v, svid, faces, inc_ptr, inc);
    if (!(dot3(n, n) > 1e-20f)) n = make_float3(0.f, 0.f, 1.f);               // tetmesh_geometry.py:57-60
    const float inv = 1.f / fmaxf(sqrtf(dot3(n, n)), 1e-12f);                    // F.normalize eps
    v_nrm[3 * size_t(a)] = n.x * inv; v_nrm[3 * size_t(a) + 1] = n.y * inv; v_nrm[3 * size_t(a) + 2] = n.z * inv;
  }
}

// h_a = d L / d (raw normal of a) = (I - n^ n^T) g_a / |n|   (0 where the fallback replaced the normal)
__global__ void surface_backward_h_kernel(const float *__restrict__ tet_v, const int32_t *__restrict__ svid, const int32_t *__restrict__ faces,
                                          const int32_t *__restrict__ inc_ptr, const int32_t *__restrict__ inc, int nsv,
                                          const float *__restrict__ g_nrm, float *__restrict__ h) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= nsv) return;
  float3 out = make_float3(0.f, 0.f, 0.f);
  const float3 n = raw_normal(a, tet_v, svid, faces, inc_ptr, inc);
  const float nn = dot3(n, n);
  if (nn > 1e-20f) {
    const float len = fmaxf(sqrtf(nn), 1e-12f), inv = 1.f / len;
    const float3 u = make_float3(n.x * inv, n.y * inv, n.z * inv), g = ld3(g_nrm, a);
    const float ug = dot3(u, g);
    out = make_float3((g.x - u.x * ug) * inv, (g.y - u.y * ug) * inv, (g.z - u.z * ug) * inv);
  }
  h[3 * size_t(a)] = out.x; h[3 * size_t(a) + 1] = out.y; h[3 * size_t(a) + 2] = out.z;
}

// grad_tet_v[svid[a]] = g_pos[a] + sum over incident faces of the face's pull on corner a
__global__ void surface_backward_kernel(const float *__restrict__ tet_v, const int32_t *__restrict__ svid, const int32_t *__restrict__ faces,
                                        const int32_t *__restrict__ inc_ptr, const int32_t *__restrict__ inc, int nsv,
                                        const float *__restrict__ g_pos, const float *__restrict__ h, float *__restrict__ grad_tet_v) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= nsv) return;
  float3 acc = g_pos ? ld3(g_pos, a) : make_float3(0.f, 0.f, 0.f);
  if (h) {
    for (int e = inc_ptr[a]; e < inc_ptr[a + 1]; ++e) {
      const int f = inc[e] >> 2, role = inc[e] & 3;
      const int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
      const float3 v0 = ld3(tet_v, svid[i0]), v1 = ld3(tet_v, svid[i1]), v2 = ld3(tet_v, svid[i2]);
      const float3 e1 = sub3(v1, v0), e2 = sub3(v2, v0);
      const float3 G = add3(add3(ld3(h, i0), ld3(h, i1)), ld3(h, i2));        // the face normal was splatted to its 3 vertices
      const float3 d1 = cross3(e2, G), d2 = cross3(G, e1);                    // dL/dv1, dL/dv2
      if (role == 1) acc = add3(acc, d1);
      else if (role == 2) acc = add3(acc, d2);
      else acc = sub3(acc, add3(d1, d2));
    }
  }
  const size_t o = 3 * size_t(svid[a]);
  grad_tet_v[o] = acc.x; grad_tet_v[o + 1] = acc.y; grad_tet_v[o + 2] = acc.z;
}

int sfail(tsb_surface_t s, int code, const std::string &msg) {
  if (s) s->err = msg; else g_surface_err = msg;
  return code;
}

template <class T>
bool up(std::vector<void *> &allocs, const std::vector<T> &v, T **out) {
  void *d = nullptr;
  if (cudaMalloc(&d, std::max<size_t>(v.size(), 1) * sizeof(T)) != cudaSuccess) return false;
  allocs.push_back(d);
  if (!v.empty() && cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) return false;
  *out = static_cast<T *>(d);
  return true;
}

}  // namespace

extern "C" {

int tsb_surface_create(const int32_t *surface_vid, int32_t nsv, const int32_t *surface_f, int32_t nsf, int32_t n_tet_vertices,
                       int device, tsb_surface_t *out) {
  if (!out) return sfail(nullptr, TSB_E_INVALID, "out is null");
  *out = nullptr;
  if (!surface_vid || !surface_f || nsv <= 0 || nsf <= 0 || n_tet_vertices <= 0) return sfail(nullptr, TSB_E_INVALID, "null input or non-positive size");
  std::vector<int32_t> svid(surface_vid, surface_vid + nsv), faces(surface_f, surface_f + 3 * size_t(nsf));
  {
    // one writer per gradient row: a repeated id would have two threads of surface_backward_kernel store the same row
    std::vector<uint8_t> seen(size_t(n_tet_vertices), 0);
    for (int32_t i = 0; i < nsv; ++i) {
      const int32_t v = svid[i];
      if (v < 0 || v >= n_tet_vertices) return sfail(nullptr, TSB_E_MESH, "surface_vid out of range");
      if (seen[size_t(v)]) return sfail(nullptr, TSB_E_MESH, "surface_vid repeats tet vertex " + std::to_string(v) + " (entry " + std::to_string(i) + ")");
      seen[size_t(v)] = 1;
    }
  }
  std::vector<int32_t> inc_ptr(size_t(nsv) + 1, 0), inc(3 * size_t(nsf));
  for (int32_t v : faces) {
    if (v < 0 || v >= nsv) return sfail(nullptr, TSB_E_MESH, "surface face index out of range");
    ++inc_ptr[v + 1];
  }
  for (int i = 0; i < nsv; ++i) inc_ptr[i + 1] += inc_ptr[i];
  {
    std::vector<int32_t> cur(inc_ptr.begin(), inc_ptr.end() - 1);
    for (int f = 0; f < nsf; ++f)
      for (int c = 0; c < 3; ++c) inc[cur[faces[3 * size_t(f) + c]]++] = f * 4 + c;     // ascending face id per vertex
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
    cudaGetLastError();
    return sfail(nullptr, TSB_E_CUDA, "no CUDA device (tssplat_b200 has no CPU path)");
  }
  Guard g(device);
  tsb_surface_t s = new tsb_surface_s();
  s->device = device; s->nsv = nsv; s->nsf = nsf; s->n = n_tet_vertices;
  std::vector<void *> allocs;
  std::vector<float> hz(3 * size_t(nsv), 0.f);
  if (!up(allocs, svid, &s->svid) || !up(allocs, faces, &s->faces) || !up(allocs, inc_ptr, &s->inc_ptr) || !up(allocs, inc, &s->inc) ||
      !up(allocs, hz, &s->h)) {
    for (void *p : allocs) cudaFree(p);
    delete s;
    cudaGetLastError();
    return sfail(nullptr, TSB_E_NOMEM, "device allocation failed");
  }
  *out = s;
  return TSB_OK;
}

void tsb_surface_destroy(tsb_surface_t s) {
  if (!s) return;
  Guard g(s->device);
  cudaFree(s->svid); cudaFree(s->faces); cudaFree(s->inc_ptr); cudaFree(s->inc); cudaFree(s->h);
  delete s;
}

const char *tsb_surface_last_error(tsb_surface_t s) { return s ? s->err.c_str() : g_surface_err.c_str(); }

int tsb_surface_forward(tsb_surface_t s, const float *tet_v_dev, float *v_pos_dev, float *v_nrm_dev, void *stream) {
  if (!s || !tet_v_dev) return sfail(s, TSB_E_INVALID, "null handle or tet_v");
  Guard g(s->device);
  surface_forward_kernel<<<(s->nsv + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(tet_v_dev, s->svid, s->faces, s->inc_ptr, s->inc,
                                                                                            s->nsv, v_pos_dev, v_nrm_dev);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? TSB_OK : sfail(s, TSB_E_CUDA, std::string("surface forward launch: ") + cudaGetErrorString(e));
}

int tsb_surface_backward(tsb_surface_t s, const float *tet_v_dev, const float *grad_v_pos_dev, const float *grad_v_nrm_dev,
                         float *grad_tet_v_dev, void *stream) {
  if (!s || !tet_v_dev || !grad_tet_v_dev) return sfail(s, TSB_E_INVALID, "null handle, tet_v or output");
  Guard g(s->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(grad_tet_v_dev, 0, size_t(s->n) * 3 * sizeof(float), st);      // non-surface vertices get no gradient
  const int grid = (s->nsv + 127) / 128;
  if (e == cudaSuccess && grad_v_nrm_dev) {
    surface_backward_h_kernel<<<grid, 128, 0, st>>>(tet_v_dev, s->svid, s->faces, s->inc_ptr, s->inc, s->nsv, grad_v_nrm_dev, s->h);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) {
    surface_backward_kernel<<<grid, 128, 0, st>>>(tet_v_dev, s->svid, s->faces, s->inc_ptr, s->inc, s->nsv, grad_v_pos_dev,
                                                 grad_v_nrm_dev ? s->h : nullptr, grad_tet_v_dev);
    e = cudaGetLastError();
  }
  return e == cudaSuccess ? TSB_OK : sfail(s, TSB_E_CUDA, std::string("surface backward: ") + cudaGetErrorString(e));
}

}  // extern "C"
