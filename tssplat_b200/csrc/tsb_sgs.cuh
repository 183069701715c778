// Multicolour block symmetric Gauss-Seidel preconditioner of the per-component solve (tsb_sgs.cu; tsb_pcg_enable_sgs in
// include/tssplat_b200.h; DESIGN.md section 5, "Symmetric Gauss-Seidel preconditioner").
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "tsb_solver.cuh"

namespace tsb {

constexpr int kSgsT = 1024;   // threads per CTA of the sweep (one CTA per component): 32 warps share a colour's rows

// The tables of tsb::SgsTables on the device, and the assembled matrix they index.
struct SgsParams {
  const int32_t *comp_off;    // [n_components + 1] first entry of every component in PcgParams::vert
  const int32_t *color_ptr;   // [n_components + 1]
  const int32_t *color_off;   // first sched entry of every colour of every component
  const int32_t *sched;       // [rows] entries grouped by colour
  const int32_t *lo_ptr, *hi_ptr;   // [rows + 1]
  const int2 *lo, *hi;        // (block, column position in the component)
  const float *values;        // [nnzb, 9] A
  const int32_t *crow, *col;  // the pattern (diagonal extraction)
  int32_t max_verts;          // vertices of the largest component: the sweep's shared memory is 12 max_verts bytes
};

// What one sweep launch reads and writes: z = M^-1 r on the components it does not skip, and per chunk of those the fp64
// partials of r.z (and of r.r when col_rr >= 0) at part[stride * chunk + col].  Skipped: with comp, the components whose
// st_upd is not active (after an update kernel); with tr_state, those whose radius is initialised (the radius start).
struct SgsSweep {
  const float *r;
  float *z;
  double *part;
  int32_t stride, col_rz, col_rr;
  const PcgComp *comp;
  const TrState *tr_state;
};

// On the current device: *max_verts = the most vertices a component may have, and, when max_comp_verts fits, the sweep's
// dynamic shared memory limit raised to 12 max_comp_verts bytes
cudaError_t sgs_configure(int max_comp_verts, int *max_verts);
cudaError_t launch_sgs_sweep(const PcgParams &s, const SgsParams &g, const SgsSweep &w, cudaStream_t st);
// diag_out [2, n, 3] from the diagonal blocks of g.values (orphan rows zero)
cudaError_t launch_sgs_diag(const SgsParams &g, int n, float *diag_out, cudaStream_t st);

}  // namespace tsb
