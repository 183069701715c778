// TEST INFRASTRUCTURE: host-only inspection of the product's plan builder (tsb_plan.cpp) so the CPU
// test-suite can re-enact the kernel's stream walk in numpy and compare it with the oracle without a
// GPU.  It lives beside the builder because it sets PlanConfig fields and must change with them.
// Built into tests/native/libtsb_plan_debug.so by __graft_entry__.build(); never part of
// libtssplat_b200.so.
#include <algorithm>
#include <cstring>
#include <string>

#include "../../include/tssplat_b200.h"
#include "tsb_plan.h"

struct tsbdbg_plan { tsb::HostPlan plan; tsb::PcgLists pcg; };
static thread_local std::string g_err;

extern "C" {

const char *tsbdbg_last_error() { return g_err.c_str(); }

/* The plan tsb_create would build.  ring_cells: the ring it requests (ring_slots * kCellsPerChunk; 0 = the default);
   enable_amips: emit the AMIPS rest inverses "Bt" and the tet-cell numbering "wtc0"; deterministic: emit the
   deterministic gather's lists "det_*" and "wtc0".  vh_cap, area_cap, tet_cost: 0 = the default. */
int tsbdbg_build_det(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele, int32_t nw, int32_t grid,
                     int32_t laplacian_scale, int32_t force_global, int32_t vh_cap, int32_t area_cap, float tet_cost,
                     int32_t ring_cells, int32_t enable_amips, int32_t deterministic, tsbdbg_plan **out) {
  if (!out) return TSB_E_INVALID;
  *out = nullptr;
  tsb::PlanConfig pc;
  pc.nw = nw; pc.grid = grid; pc.laplacian_scale = laplacian_scale; pc.force_global = force_global;
  pc.enable_amips = enable_amips ? 1 : 0;
  pc.deterministic = deterministic ? 1 : 0;
  if (vh_cap > 0) pc.vh_cap = vh_cap;
  if (area_cap > 0) pc.area_cap = area_cap;
  if (tet_cost > 0) pc.tet_cost = tet_cost;
  if (ring_cells > 0) pc.ring_cells = ring_cells;
  tsbdbg_plan *d = new tsbdbg_plan();
  const int rc = tsb::build_plan(rest_xyz, tets, n, nele, pc, d->plan, g_err);
  if (rc != TSB_OK) { delete d; return rc; }
  tsb::build_pcg_lists(d->plan.comp_label, d->plan.n_components, d->pcg);   // what tsb_pcg_create uploads
  *out = d;
  return TSB_OK;
}

/* tsbdbg_build_det with deterministic = 0: the entry point earlier test helpers call, so that they keep running
   against this library */
int tsbdbg_build_ex(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele, int32_t nw, int32_t grid,
                    int32_t laplacian_scale, int32_t force_global, int32_t vh_cap, int32_t area_cap, float tet_cost,
                    int32_t ring_cells, int32_t enable_amips, tsbdbg_plan **out) {
  return tsbdbg_build_det(rest_xyz, tets, n, nele, nw, grid, laplacian_scale, force_global, vh_cap, area_cap, tet_cost,
                          ring_cells, enable_amips, 0, out);
}

/* name ->(pointer, element count, element bytes); TSB_E_INVALID for an unknown name */
int tsbdbg_array(tsbdbg_plan *d, const char *name, const void **ptr, int64_t *count, int32_t *elem_bytes) {
  if (!d || !name || !ptr || !count || !elem_bytes) return TSB_E_INVALID;
  const tsb::HostPlan &P = d->plan;
  const std::string k(name);
#define ARR(nm, vec, eb) if (k == nm) { *ptr = (vec).data(); *count = int64_t((vec).size()) * int64_t(sizeof((vec)[0])) / (eb); *elem_bytes = (eb); return TSB_OK; }
  ARR("stream", P.stream, 1) ARR("X4", P.X4, 4) ARR("vlist", P.vlist, 4) ARR("segs", P.segs, 4) ARR("cta_seg", P.cta_seg, 4)
  ARR("wdesc", P.wdesc, 4) ARR("wseg", P.wseg, 2) ARR("orphans", P.orphans, 4) ARR("pos16", P.pos16, 2) ARR("pos_gid", P.pos_gid, 4)
  ARR("Bt", P.Bt, 4) ARR("wtc0", P.wtc0, 4)
  ARR("det_rowptr", P.det_rowptr, 4) ARR("det_vert", P.det_vert, 4) ARR("det_ent", P.det_ent, 4)
  ARR("det_comp_row", P.det_comp_row, 4) ARR("det_chunk", P.det_chunk, 4)
  ARR("comp_seg", P.comp_seg, 4) ARR("comp_first_vertex", P.comp_first_vertex, 4) ARR("comp_ntets", P.comp_ntets, 4)
  ARR("comp_label", P.comp_label, 4) ARR("pcg_vert", d->pcg.vert, 4) ARR("pcg_comp_off", d->pcg.comp_off, 4)
  ARR("pcg_chunk", d->pcg.chunk, 4) ARR("pcg_comp_chunk", d->pcg.comp_chunk, 4)
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

/* The block pattern and tet tables tsb_hessian_create uploads (tsb::build_hessian_pattern, tsb::build_tet_tables);
   arrays through tsbdbg_hess_array: "crow", "col", "w", "tblk", "inc_ptr", "inc", "B", "comp_label" */
struct tsbdbg_hess { tsb::HessPattern H; tsb::TetTables T; };

int tsbdbg_hess_build(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele, int32_t laplacian_scale,
                      tsbdbg_hess **out, int64_t *nnzb) {
  if (!out || !nnzb) return TSB_E_INVALID;
  *out = nullptr;
  tsbdbg_hess *d = new tsbdbg_hess();
  int rc = tsb::build_hessian_pattern(rest_xyz, tets, n, nele, laplacian_scale, d->H, g_err);
  if (rc == TSB_OK) rc = tsb::build_tet_tables(rest_xyz, tets, n, nele, nullptr, d->T, g_err);
  if (rc != TSB_OK) { delete d; return rc; }
  *nnzb = d->H.nnzb;
  *out = d;
  return TSB_OK;
}

int tsbdbg_hess_array(tsbdbg_hess *d, const char *name, const void **ptr, int64_t *count) {
  if (!d || !name || !ptr || !count) return TSB_E_INVALID;
  const tsb::HessPattern &H = d->H;
  const std::string k(name);
#define ARR(nm, vec) if (k == nm) { *ptr = (vec).data(); *count = int64_t((vec).size()); return TSB_OK; }
  ARR("crow", H.crow) ARR("col", H.col) ARR("w", H.w) ARR("tblk", H.tblk) ARR("inc_ptr", d->T.inc_ptr) ARR("inc", d->T.inc)
  ARR("B", d->T.B) ARR("comp_label", H.comp_label)
#undef ARR
  return TSB_E_INVALID;
}

void tsbdbg_hess_free(tsbdbg_hess *d) { delete d; }

/* The multicolour Gauss-Seidel tables tsb_pcg_enable_sgs builds (tsb::build_sgs_tables) over the pattern and the solver's
   vertex lists of the mesh, with nth host threads (0: the default); arrays through tsbdbg_sgs_array: "color", "lo_ptr",
   "hi_ptr", "lo", "hi", "sched", "color_ptr", "color_off", and the lists "crow", "col", "vert", "comp_off" it was built
   from */
struct tsbdbg_sgs { tsb::HessPattern H; tsb::PcgLists L; tsb::SgsTables T; };

int tsbdbg_sgs_build(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele, int32_t laplacian_scale, int32_t nth,
                     tsbdbg_sgs **out, int32_t *n_colors) {
  if (!out || !n_colors) return TSB_E_INVALID;
  *out = nullptr;
  tsbdbg_sgs *d = new tsbdbg_sgs();
  int rc = tsb::build_hessian_pattern(rest_xyz, tets, n, nele, laplacian_scale, d->H, g_err);
  if (rc == TSB_OK) {
    int32_t S = 0;
    for (const int32_t c : d->H.comp_label) S = std::max(S, c + 1);
    tsb::build_pcg_lists(d->H.comp_label, S, d->L);
    rc = tsb::build_sgs_tables(d->H.crow, d->H.col, d->L, nth, d->T, g_err);
  }
  if (rc != TSB_OK) { delete d; return rc; }
  *n_colors = d->T.n_colors;
  *out = d;
  return TSB_OK;
}

int tsbdbg_sgs_array(tsbdbg_sgs *d, const char *name, const void **ptr, int64_t *count) {
  if (!d || !name || !ptr || !count) return TSB_E_INVALID;
  const tsb::SgsTables &T = d->T;
  const std::string k(name);
#define ARR(nm, vec) if (k == nm) { *ptr = (vec).data(); *count = int64_t((vec).size()); return TSB_OK; }
  ARR("color", T.color) ARR("lo_ptr", T.lo_ptr) ARR("hi_ptr", T.hi_ptr) ARR("lo", T.lo) ARR("hi", T.hi) ARR("sched", T.sched)
  ARR("color_ptr", T.color_ptr) ARR("color_off", T.color_off)
  ARR("crow", d->H.crow) ARR("col", d->H.col) ARR("vert", d->L.vert) ARR("comp_off", d->L.comp_off)
#undef ARR
  return TSB_E_INVALID;
}

void tsbdbg_sgs_free(tsbdbg_sgs *d) { delete d; }

/* The coarse-space tables tsb_pcg_enable_coarse builds (tsb::build_coarse_tables) over build_tet_tables and the solver's
   vertex lists of the mesh; arrays through tsbdbg_coarse_array: "tet", "tets", "B", "tchunk", "comp_tchunk", "Y", "S",
   and the lists "vert", "comp_off", "comp_label" it was built from */
struct tsbdbg_coarse { tsb::HessPattern H; tsb::PcgLists L; tsb::TetTables T; tsb::CoarseTables C; };

int tsbdbg_coarse_build(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele, tsbdbg_coarse **out,
                        int32_t *n_components) {
  if (!out || !n_components) return TSB_E_INVALID;
  *out = nullptr;
  tsbdbg_coarse *d = new tsbdbg_coarse();
  int rc = tsb::build_hessian_pattern(rest_xyz, tets, n, nele, 0, d->H, g_err);
  int32_t S = 0;
  if (rc == TSB_OK) {
    for (const int32_t c : d->H.comp_label) S = std::max(S, c + 1);
    tsb::build_pcg_lists(d->H.comp_label, S, d->L);
    rc = tsb::build_tet_tables(rest_xyz, tets, n, nele, &d->H.comp_label, d->T, g_err);
  }
  if (rc != TSB_OK) { delete d; return rc; }
  tsb::build_coarse_tables(rest_xyz, d->T, d->H.comp_label, d->L, d->C);
  *n_components = S;
  *out = d;
  return TSB_OK;
}

int tsbdbg_coarse_array(tsbdbg_coarse *d, const char *name, const void **ptr, int64_t *count) {
  if (!d || !name || !ptr || !count) return TSB_E_INVALID;
  const tsb::CoarseTables &C = d->C;
  const std::string k(name);
#define ARR(nm, vec) if (k == nm) { *ptr = (vec).data(); *count = int64_t((vec).size()); return TSB_OK; }
  ARR("tet", C.tet) ARR("tets", C.tets) ARR("B", C.B) ARR("tchunk", C.tchunk) ARR("comp_tchunk", C.comp_tchunk) ARR("Y", C.Y)
  ARR("S", C.S) ARR("vert", d->L.vert) ARR("comp_off", d->L.comp_off) ARR("comp_label", d->H.comp_label)
#undef ARR
  return TSB_E_INVALID;
}

void tsbdbg_coarse_free(tsbdbg_coarse *d) { delete d; }

}  // extern "C"
