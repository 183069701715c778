// Device-side tables and launchers of the per-component Newton-CG solver (tsb_solver.cu), used by tsb_capi.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/tssplat_b200.h"
#include "tsb_plan.h"

namespace tsb {

constexpr int32_t kPcgActive = -1;   // internal status of a component that is still iterating (reported as MAXITER)

// State of one component.  Every field has one writing kernel (its component's first chunk) and is only read by other
// kernels, so no launch reads a value another CTA of the same launch may be writing; the per-chunk partial table
// follows the same rule column by column (tsb_solver.cu).  64 bytes.
struct PcgComp {
  double rz;        // r.z of the current residual          (dir writes, update reads)
  double rz_prev;   // r.z before the last update           (update writes, dir reads)
  double bb;        // |b_c|^2                              (first dir writes)
  double rr;        // |r_c|^2 of the current residual      (dir writes)
  double dHd;       // sum of alpha^2 p^T H p               (first dir clears, update adds)
  int32_t st_dir;   // status after the last dir kernel     (dir writes; curv and update read)
  int32_t st_upd;   // status after the last update kernel  (update writes; dir reads)
  int32_t idle;     // 1: already stopped before the last update, so its p is already 0   (update writes; dir reads)
  int32_t n_hvp;    // products in which it was active      (first dir clears, update writes)
  int32_t pad[2];
};
static_assert(sizeof(PcgComp) == 64, "PcgComp must be 64 bytes");

struct PcgParams {
  const int32_t *vert;         // [rows] vertex ids grouped by component (PcgLists::vert)
  const int32_t *comp_chunk;   // [n_components + 1] first chunk of every component
  const int32_t *chunk;        // [3 * n_chunks] (component, begin, end)
  const int32_t *orphans;      // the handle's list of vertices no tet references
  int32_t n_chunks, n_components, n_orphans, n;
  float *r, *z, *p, *Hp;       // [n, 3]
  float *pinv;                 // [n, 6] inverse preconditioner blocks: xx yy zz yz xz xy
  double *part;                // [n_chunks, 3] per-chunk partial sums: p.Hp (or b.d), r.z, r.r
  PcgComp *comp;               // [n_components]
  int32_t *active;             // [1] components still active (pcg_count_kernel)
};

cudaError_t launch_pcg_blocks(const PcgParams &s, const float *diag, float rel_floor, float *inv_out, cudaStream_t st);
// r = b, z = P r, d = 0 and the first direction; leaves every component ACTIVE or ZERO_RHS
cudaError_t launch_pcg_begin(const PcgParams &s, const float *b, float *d, cudaStream_t st);
// after Hp = H p of iteration `iter` (0-based) is complete on the stream: curvature, update and next direction
cudaError_t launch_pcg_step(const PcgParams &s, float *d, int iter, float rtol, cudaStream_t st);
cudaError_t launch_pcg_count(const PcgParams &s, cudaStream_t st);
cudaError_t launch_pcg_records(const PcgParams &s, const float *b, const float *d, tsb_pcg_sphere_t *out, cudaStream_t st);
cudaError_t launch_sphere_axpy(const PcgParams &s, const float *x, const float *a, const float *d, float *out, cudaStream_t st);

}  // namespace tsb
