// TEST INFRASTRUCTURE: host-only inspection of the product's plan builder (tsb_plan.cpp) so the CPU
// test-suite can re-enact the kernel's stream walk in numpy and compare it with the oracle without a
// GPU.  It lives beside the builder because it sets PlanConfig fields and must change with them.
// Built into tests/native/libtsb_plan_debug.so by __graft_entry__.build(); never part of
// libtssplat_b200.so.
#include <cstring>
#include <string>

#include "../../include/tssplat_b200.h"
#include "tsb_plan.h"

struct tsbdbg_plan { tsb::HostPlan plan; };
static thread_local std::string g_err;

extern "C" {

const char *tsbdbg_last_error() { return g_err.c_str(); }

int tsbdbg_build(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele, int32_t nw, int32_t grid,
                 int32_t laplacian_scale, int32_t force_global, int32_t vh_cap, int32_t area_cap, float tet_cost,
                 tsbdbg_plan **out) {
  if (!out) return TSB_E_INVALID;
  *out = nullptr;
  tsb::PlanConfig pc;
  pc.nw = nw; pc.grid = grid; pc.laplacian_scale = laplacian_scale; pc.force_global = force_global;
  if (vh_cap > 0) pc.vh_cap = vh_cap;
  if (area_cap > 0) pc.area_cap = area_cap;
  if (tet_cost > 0) pc.tet_cost = tet_cost;
  tsbdbg_plan *d = new tsbdbg_plan();
  const int rc = tsb::build_plan(rest_xyz, tets, n, nele, pc, d->plan, g_err);
  if (rc != TSB_OK) { delete d; return rc; }
  *out = d;
  return TSB_OK;
}

/* name -> (pointer, element count, element bytes); TSB_E_INVALID for an unknown name */
int tsbdbg_array(tsbdbg_plan *d, const char *name, const void **ptr, int64_t *count, int32_t *elem_bytes) {
  if (!d || !name || !ptr || !count || !elem_bytes) return TSB_E_INVALID;
  const tsb::HostPlan &P = d->plan;
  const std::string k(name);
#define ARR(nm, vec, eb) if (k == nm) { *ptr = (vec).data(); *count = int64_t((vec).size()) * int64_t(sizeof((vec)[0])) / (eb); *elem_bytes = (eb); return TSB_OK; }
  ARR("stream", P.stream, 1) ARR("X4", P.X4, 4) ARR("vlist", P.vlist, 4) ARR("segs", P.segs, 4) ARR("cta_seg", P.cta_seg, 4)
  ARR("wdesc", P.wdesc, 4) ARR("wseg", P.wseg, 2) ARR("orphans", P.orphans, 4) ARR("pos16", P.pos16, 2) ARR("pos_gid", P.pos_gid, 4)
#undef ARR
  return TSB_E_INVALID;
}

int tsbdbg_scalars(tsbdbg_plan *d, int64_t *out16) {   /* out16: 20 entries */
  if (!d || !out16) return TSB_E_INVALID;
  const tsb::HostPlan &P = d->plan;
  const int64_t v[20] = {P.n, P.nele, P.n_components, P.n_boundary_faces, P.laplacian_scale, P.mode_global, P.nw, P.grid,
                         P.vh, P.area_verts, P.max_comp_verts, P.contiguous, P.nnz, P.nnz_padded, P.n_rb, P.n_tetcells,
                         P.gather_wavefronts[0], P.gather_wavefronts[1], P.tet_wavefronts[0], P.tet_wavefronts[1]};
  std::memcpy(out16, v, sizeof(v));
  return TSB_OK;
}

void tsbdbg_free(tsbdbg_plan *d) { delete d; }

}  // extern "C"
