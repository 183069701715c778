// Device-side parameter block shared by tsb_kernels.cu (kernels) and tsb_capi.cu (C ABI).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/tssplat_b200.h"
#include "tsb_plan.h"

namespace tsb {

// What one warp saw of one segment (SPH instantiation): its lanes' energy partials in fp64 (smoothness not yet
// halved), the smallest J of its real tets (+inf: none) and how many of them have J < 0.  32 bytes.
struct __align__(16) SphRec {
  double smooth, barrier, amips;
  float min_J;
  int32_t n_inverted;
};
static_assert(sizeof(SphRec) == 32, "SphRec must be 32 bytes");

// What one CTA saw of one segment in a line search (LINE instantiation), in fp64: v[k] = barrier change at alpha_k,
// v[8 + k] = AMIPS change, v[16] = u^T M d and v[17] = d^T M d over the segment's rows, v[18] = the smallest first
// root of a tet's det F along d (+inf: none).  Segment s's record lies at byte s * nw * 32 of the sph_rec array (nw
// SphRec slots per segment, >= 256 bytes), so the line search needs no device memory of its own.  line_fold_kernel
// overwrites the record of a component's first segment with the component's sums.
constexpr int kLineMaxAlpha = TSB_LINE_MAX_ALPHA;
constexpr int kLineVals = 2 * kLineMaxAlpha + 3;
struct LineRec {
  double v[kLineVals];
};
static_assert(sizeof(LineRec) <= 8 * sizeof(SphRec), "a LineRec must fit the SphRec slots of one segment");
__host__ __device__ inline LineRec *line_rec(SphRec *base, int s, int nw) {
  return reinterpret_cast<LineRec *>(reinterpret_cast<unsigned char *>(base) + size_t(s) * size_t(nw) * sizeof(SphRec));
}

struct KParams {
  // plan (read-only, built once by tsb_create)
  const unsigned char *stream;  // per-warp byte streams (operator rows + tet blocks)
  const float4 *X4;             // rest positions (STAGED: component-major; GLOBAL: by vertex id, .w = reference vertex)
  const int32_t *vlist;         // STAGED: global vertex id per staged vertex (used when a component is not contiguous)
  const uint16_t *pos16;        // STAGED: staging position per staged vertex (bank-aware placement)
  const int32_t *pos_gid;       // STAGED: global vertex id per staging position
  const SegHdr *segs;
  const int2 *cta_seg;          // per CTA: [first segment, one past last)
  const uint2 *wdesc;           // per (CTA, warp): (stream offset / 16, stream bytes)
  const ushort2 *wseg;          // per (segment, warp): (row blocks, tet blocks)
  const float4 *Bt;             // AMIPS: rest inverses per streamed tet ([cell][row][slot] float4), or nullptr
  const int32_t *wtc0;          // AMIPS: first tet cell of every (segment, warp)
  const int32_t *orphans;       // vertices without tets
  int32_t n_orphans;
  int32_t n_components;
  // per-handle scratch (self-resetting)
  unsigned int *done;           // [n_components] warps that have stored their rows of a component
  double *cta_energy;           // [4*grid] (smooth, barrier, amips, 0) partials per CTA; a NaN-payload sentinel = "not written yet"
  float4 *u4g, *x4g;            // GLOBAL mode: displacement / position per vertex (written by the pre-pass)
  // per launch
  const float *x;               // [3n]
  float *grad;                  // [3n] or nullptr (energy only)
  float *energy_out;            // [3]: total, smooth, barrier
  const float *gradH_dev;       // optional device scalar
  float c1, c2, c3, gradH;      // c3: AMIPS coefficient (0 = term off)
  int32_t order;                // 2 or 4
  int32_t energy4;              // energy_out has 4 entries (total, smooth, barrier, amips)
  int32_t n;                    // vertices
  int32_t vh;                   // STAGED: half-buffer capacity in vertices
  int32_t ring_bytes;           // per-warp ring size = slots * cells_per_chunk cells
  int32_t cells_per_chunk;      // cells per TMA bulk copy (= per ring slot)
  int32_t ring_slots;
  int32_t stage_bytes;          // STAGED: bytes of the staging area at the start of shared memory
  // deterministic gradient only (tsb_options_t.deterministic): per-handle scratch the DET instantiation fills and
  // det_gather_kernel consumes.  Tet slot (wtc0 + tc) * (tets per cell) + lane * TPL + t (tsb_plan.h).
  float4 *det_scratch;          // [3 * slots] corner vectors of a contributing tet: (c0.xyz, c1.x) (c1.yz, c2.xy) (c2.z, c3.xyz)
  unsigned long long *det_ballot;   // [tet cells] bit t * 32 + lane: the tet in slot lane * TPL + t contributed
  unsigned int *det_flag;       // [n_components] nonzero: a tet of the component contributed (the gather clears it)
  // per-sphere statistics only (the SPH instantiation, tsb_energy_grad_spheres): one record per (segment, warp)
  SphRec *sph_rec;              // [n_segments * nw], rewritten by every SPH launch, read by sphere_fold_kernel
  // Hessian-vector product only (the HVP instantiations, tsb_hvp / tsb_hvp_ex): grad receives gradH H(x) v, energy_out
  // (may be nullptr) v^T H v as (c1 vMv + c2 vHbv + c3 vHav, vMv, vHbv[, vHav when energy4])
  const float *v;               // [3n] direction
  // line search only (the LINE instantiations, tsb_line_search): v is the direction d, grad and energy_out are nullptr,
  // and the per-segment records (LineRec) are written over sph_rec
  const float *alpha;           // [n_alpha] step sizes, read on the device
  int32_t n_alpha;              // 1..kLineMaxAlpha
  // Hessian diagonal only (the DIAG instantiations, tsb_hess_diag): grad receives the per-vertex 3x3 diagonal blocks,
  // (H_xx, H_yy, H_zz) in plane 0 and (H_yz, H_xz, H_xy) in plane 1 (grad + 3n).  DET: one launch per plane, grad points
  // at that plane and diag_plane selects it (a tet slot holds one plane of its four corners)
  int32_t diag_plane;
#ifdef TSB_TRACE
  unsigned long long *trace;    // profiling build only: [grid][kTraceSlots] phase stamps
#endif
};
constexpr int kTraceSlots = 16 + kMaxWarps;   // profiling build: 16 phase stamps of thread 0, then one per warp

struct LaunchConfig {
  int nw;          // warps per CTA (8 or 16)
  int grid;        // persistent CTAs
  int smem_bytes;  // dynamic shared memory
  int global;      // GLOBAL mode
  int amips;       // launch the AMIPS-capable instantiation
  int det;         // launch the deterministic instantiation (tets store their corners instead of adding them)
  int sph;         // launch the SPH instantiation (it also writes the per-(segment, warp) sphere records)
  int hvp;         // launch the HVP instantiation (Hessian-vector product; never with sph)
  int line;        // launch the LINE instantiation (line search; combines with amips only)
  int diag;        // launch the DIAG instantiation (Hessian diagonal blocks; combines with amips and det only)
};

// sphere_fold_kernel's inputs (HostPlan::comp_*, uploaded, and the records of the SPH launch before it).
struct SphParams {
  const SphRec *rec;
  const int32_t *comp_seg;          // [n_components + 1] first segment of every component
  const int32_t *comp_first_vertex; // [n_components]
  const int32_t *comp_ntets;        // [n_components]
  int32_t n_components;
  int32_t nw;
};

// The deterministic gather's plan (HostPlan::det_*, uploaded) and the scratch it shares with the energy kernel.
struct DetParams {
  const int32_t *rowptr, *vert, *comp_row;
  const uint32_t *ent;              // slot * 4 + corner
  const int2 *chunk;                // (component, first row) of every CTA
  const float4 *scratch;
  const unsigned long long *ballot;
  unsigned int *flag;
  int32_t n_chunks;
  int32_t tpl_log;                  // log2(tets per lane): 1 STAGED, 0 GLOBAL
};

// Dynamic shared memory the kernel needs for a configuration (ring_slots chunks of cells_per_chunk cells per warp).
int energy_ring_bytes(int ring_slots, int cells_per_chunk, bool global);
int energy_smem_bytes(int nw, int ring_slots, int cells_per_chunk, int area_verts, bool global);
constexpr unsigned long long kEnergySentinel = 0x7FF8F00DBAADC0DEull;   // initial value of cta_energy
// Max co-resident CTAs per SM for a configuration (0 if it does not fit): the minimum over every instantiation a handle
// may launch (AMIPS ones when amips, deterministic ones when det, each with and without the sphere records, and the
// Hessian-vector product, line search and Hessian diagonal ones); also opts them in to the smem size.
cudaError_t energy_occupancy(int nw, int smem_bytes, bool global, bool amips, bool det, int *ctas_per_sm);
cudaError_t launch_energy_grad(const KParams &p, const LaunchConfig &lc, cudaStream_t stream);
// grad[v] += the active corner vectors of v's list, in list order, for every flagged component (after a DET launch).
cudaError_t launch_det_gather(const DetParams &d, float *grad, cudaStream_t stream);
// One tsb_sphere_stats_t per component from the records of the SPH launch before it on the same stream.
cudaError_t launch_sphere_fold(const SphParams &sp, tsb_sphere_stats_t *out, cudaStream_t stream);
// After a LINE launch on the same stream: per-component sums of its records (in place, and to the optional per-sphere
// outputs), then their fixed-order total to delta_out [n_alpha][4] and the optional step_out [1].
cudaError_t launch_line_fold(const SphParams &sp, const float *alpha, int n_alpha, float c1, float c2, float c3,
                             float *delta_out, float *step_out, float *sphere_delta_out, float *sphere_step_out,
                             cudaStream_t stream);

cudaError_t launch_scale(const float *g, int64_t count, float gradH, const float *gradH_dev, float *out, cudaStream_t s);
cudaError_t launch_grad_limit(float *g, int64_t count, float thr, float s, float *work4, cudaStream_t st);
cudaError_t launch_adam_uniform(float *p, const float *grad, float *g1, float *g2, int64_t count, double lr,
                                double b1, double b2, int step, double grad_limit, float *work4, cudaStream_t st);

}  // namespace tsb
