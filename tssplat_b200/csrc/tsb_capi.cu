// C ABI (include/tssplat_b200.h) over the plan builder and the sm_90a kernels.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/tssplat_b200.h"
#include "tsb_hessian.cuh"
#include "tsb_kernels.cuh"
#include "tsb_lbfgs.cuh"
#include "tsb_plan.h"
#include "tsb_psd.cuh"
#include "tsb_sgs.cuh"
#include "tsb_solver.cuh"

static_assert(sizeof(tsb_sphere_stats_t) == 40, "tsb_sphere_stats_t must be 40 bytes");
static_assert(sizeof(tsb_pcg_sphere_t) == 32, "tsb_pcg_sphere_t must be 32 bytes");
static_assert(sizeof(tsb_newton_options_t) == 64, "tsb_newton_options_t must be 64 bytes");
static_assert(sizeof(tsb_newton_sphere_t) == 64, "tsb_newton_sphere_t must be 64 bytes");
static_assert(sizeof(tsb_newton_tr_options_t) == 64, "tsb_newton_tr_options_t must be 64 bytes");
static_assert(sizeof(tsb_newton_tr_sphere_t) == 64, "tsb_newton_tr_sphere_t must be 64 bytes");
static_assert(sizeof(tsb_newton_backtrack_t) == 32, "tsb_newton_backtrack_t must be 32 bytes");
static_assert(sizeof(tsb_newton_lbfgs_options_t) == 64, "tsb_newton_lbfgs_options_t must be 64 bytes");
static_assert(sizeof(tsb_newton_lbfgs_sphere_t) == 64, "tsb_newton_lbfgs_sphere_t must be 64 bytes");

struct tsb_handle_s {
  int device = 0;
  tsb::KParams kp{};
  tsb::LaunchConfig lc{};
  // tsb_energy_grad_host: calls alternate between two internal streams, each running upload -> kernel ->
  // download on its own staging buffers; only the kernels are ordered across the two (ev_run), so call
  // i+1's upload overlaps call i's kernel and download.  (A third stream for the downloads, or one stream per
  // stage, costs more CPU time per call in the driver than the extra overlap saves.)
  float *stage_x[2] = {nullptr, nullptr}, *stage_grad[2] = {nullptr, nullptr}, *stage_energy[2] = {nullptr, nullptr};
  cudaStream_t s_pipe[2] = {nullptr, nullptr};
  cudaEvent_t ev_run[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
  unsigned host_calls = 0;
  bool amips = false;
  bool det = false;             // deterministic gradient: DET energy kernel + det_gather_kernel
  int32_t lap_scale = 0;        // tsb_options_t.laplacian_scale (tsb_hessian_create rebuilds the operator rows)
  tsb::DetParams dp{};
  tsb::SphParams sp{};          // per-sphere statistics: the fold's tables (records: kp.sph_rec)
  tsb_info_t info{};
  std::vector<int32_t> comp_label;   // host only: component of every vertex (-1: no tet), for tsb_pcg_create
  std::vector<void *> allocs;
  std::string err;
};

struct tsb_pcg_s {
  tsb_handle_t h = nullptr;
  int device = 0;                    // the handle's device, kept so that destroying never reads the handle
  tsb::PcgParams P{};
  int64_t device_bytes = 0;
  int32_t *active_host = nullptr;    // pinned: the "components still active" count of check_every > 0
  cudaEvent_t ev = nullptr;
  bool psd = false;                  // tsb_pcg_enable_psd: the solve multiplies by the projected Hessian
  tsb::PsdParams Q{};
  tsb::TrComp *tr = nullptr;         // [n_components] trust-region recurrences (allocated by the first tsb_pcg_solve_tr)
  tsb_hessian_t sgs = nullptr;       // tsb_pcg_enable_sgs: the Hessian workspace that assembles A, and the sweep's tables
  tsb::SgsParams G{};
  float *sgs_values = nullptr;       // [9 nnzb] A, written by tsb_pcg_set_matrix
  int32_t *sgs_color = nullptr;      // [n]
  int32_t sgs_n_colors = 0;
  bool coarse = false;               // tsb_pcg_enable_coarse: the two-level preconditioner with the affine coarse space
  tsb::CoarseParams co{};
  std::vector<void *> allocs;
  std::string err;
};

struct tsb_newton_s {
  tsb_pcg_t s = nullptr;
  int device = 0;                    // the handle's device, kept so that destroying never reads the solver workspace
                                     // (a garbage collector may free the handle and workspaces in any order)
  tsb::NewtonParams W{};
  float *energy = nullptr;           // [4] energies of the gradient launch (not reported)
  float *delta = nullptr;            // [TSB_LINE_MAX_ALPHA][4] the line search's totals (not reported)
  double *prox_part = nullptr;       // [chunks] d.(x - y) partials of tsb_newton_prox_step (allocated by its first call)
  tsb::TrState *tr_state = nullptr;  // [n_components] trust-region radius state (allocated by the first tsb_newton_tr_step)
  float *tr_radius = nullptr;        // [n_components] its fp32 radius, handed to tsb_pcg_solve_tr
  tsb::LbfgsParams lb{};             // L-BFGS history and state (allocated by the first tsb_newton_lbfgs_step; lb.m = 0 before)
  int64_t device_bytes = 0;
  std::vector<void *> allocs;
  std::string err;
};

struct tsb_hessian_s {
  tsb_pcg_t s = nullptr;
  int device = 0;                    // the handle's device, kept so that destroying never reads the solver workspace
  bool psd = false;                  // the solver workspace's mode at creation
  tsb::HessParams P{};
  int32_t *crow = nullptr, *col = nullptr;
  int64_t nnzb = 0;
  int64_t device_bytes = 0;
  std::vector<void *> allocs;
  std::string err;
};

namespace {

// What *_last_error reports for a null object: the message of the last failed create of that kind on this thread
template <class O>
std::string &create_err() {
  thread_local std::string msg;
  return msg;
}

struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int d) : dev(d) {
    if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
    if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
  }
  int dev;
  ~DeviceGuard() { if (prev >= 0 && prev != dev) cudaSetDevice(prev); }
};

// device that owns a device pointer (falls back to the current device)
int device_of(const void *p) {
  cudaPointerAttributes a{};
  if (p && cudaPointerGetAttributes(&a, p) == cudaSuccess && a.type == cudaMemoryTypeDevice) return a.device;
  cudaGetLastError();
  int d = 0;
  cudaGetDevice(&d);
  return d;
}

// The error path of every object kind (tsb_handle_t and the workspaces): the message goes to the object, or for a null
// object to its kind's creation error.
template <class O>
int fail(O *o, int code, const std::string &msg) {
  (o ? o->err : create_err<O>()) = msg;
  return code;
}

int64_t &device_bytes(tsb_handle_t h) { return h->info.device_bytes; }
template <class W>
int64_t &device_bytes(W *w) { return w->device_bytes; }

// what a failed initialisation of a new device array reports: the handle names the call
std::string init_error(tsb_handle_t, bool copy) { return copy ? "cudaMemcpy: " : "cudaMemset: "; }
template <class W>
std::string init_error(W *, bool) { return "workspace initialisation: "; }

// A device array of max(elems, n_src) elements of T owned by o: counted in its device bytes, freed by its destroy.  It
// holds src[0, n_src) when src is set (the rest uninitialised), else zeros when zero is set, else whatever was there.
// out is the kernel's typed view of the data (e.g. float4 over 4 floats).
template <class O, class D, class T = D>
int device_array(O *o, D *&out, size_t elems, const T *src = nullptr, size_t n_src = 0, bool zero = true) {
  const size_t bytes = std::max(elems, n_src) * sizeof(T);
  void *d = nullptr;
  cudaError_t e = cudaMalloc(&d, bytes);
  if (e != cudaSuccess) return fail(o, TSB_E_NOMEM, std::string("cudaMalloc: ") + cudaGetErrorString(e));
  o->allocs.push_back(d);
  device_bytes(o) += int64_t(bytes);
  if (src && n_src) e = cudaMemcpy(d, src, n_src * sizeof(T), cudaMemcpyHostToDevice);
  else if (!src && zero) e = cudaMemset(d, 0, bytes);
  if (e != cudaSuccess) return fail(o, TSB_E_CUDA, init_error(o, src != nullptr) + cudaGetErrorString(e));
  out = static_cast<D *>(d);
  return TSB_OK;
}

// Marks o's allocations and device bytes; unless commit() is called, going out of scope rolls them back.  With destroy
// (a create), it destroys the new object instead, keeping its message as the creation error.
template <class O>
class Rollback {
 public:
  explicit Rollback(O *o, void (*destroy)(O *) = nullptr)
      : o_(o), destroy_(destroy), allocs_(o->allocs.size()), bytes_(device_bytes(o)) {}
  ~Rollback() {
    if (committed_) return;
    if (destroy_) {
      create_err<O>() = o_->err;
      destroy_(o_);
      return;
    }
    for (size_t k = allocs_; k < o_->allocs.size(); ++k) cudaFree(o_->allocs[k]);
    o_->allocs.resize(allocs_);
    device_bytes(o_) = bytes_;
  }
  void commit() { committed_ = true; }

 private:
  O *o_;
  void (*destroy_)(O *);
  size_t allocs_;
  int64_t bytes_;
  bool committed_ = false;
};

// TSB_OK unless st is being captured, which is refused with `refusal`.  The legacy stream cannot be queried while another
// stream is being captured, so that counts as a capture too; any other stream that cannot be queried is TSB_E_CUDA.
template <class O>
int refuse_capture(O *o, cudaStream_t st, const char *refusal) {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  const bool queried = cudaStreamIsCapturing(st, &cap) == cudaSuccess;
  if (st == cudaStreamLegacy) {
    if (queried && cap == cudaStreamCaptureStatusNone) return TSB_OK;
    cudaGetLastError();
    return fail(o, TSB_E_INVALID, refusal);
  }
  if (!queried) { cudaGetLastError(); return fail(o, TSB_E_CUDA, "cannot query the stream"); }
  return cap == cudaStreamCaptureStatusNone ? TSB_OK : fail(o, TSB_E_INVALID, refusal);
}

// Device array of a workspace that a call allocates on its first use, of max(elems, 1) elements (zero: cleared on st).
// Nothing happens once *out is set; on a stream being captured nothing is allocated and the call is refused with `refusal`.
template <class T, class W>
int alloc_once(W *s, size_t elems, T **out, cudaStream_t st, const char *refusal, bool zero = false) {
  if (*out) return TSB_OK;
  int rc = refuse_capture(s, st, refusal);
  if (rc == TSB_OK) rc = device_array(s, *out, std::max<size_t>(elems, 1), static_cast<const T *>(nullptr), 0, false);
  if (rc != TSB_OK || !zero) return rc;
  const cudaError_t e = cudaMemsetAsync(*out, 0, std::max<size_t>(elems, 1) * sizeof(T), st);
  if (e != cudaSuccess) {
    *out = nullptr;
    return fail(s, TSB_E_CUDA, std::string("cudaMemsetAsync: ") + cudaGetErrorString(e));
  }
  return TSB_OK;
}

// The rules of a tsb_terms_t: the barrier order, AMIPS only on a handle created with it, and for the projected Hessian
// (psd) weights >= 0 (the projection multiplies by c2 and c3, so it is only the projection of the weighted sum for
// weights >= 0).  Returns the message of the first rule broken, or null.
const char *check_terms(tsb_handle_t h, bool psd, const tsb_terms_t &t) {
  if (t.order != 2 && t.order != 4) return "order must be 2 or 4";
  if (t.c3 != 0.f && !h->amips) return "c3 != 0 needs a handle created with tsb_options_t.enable_amips = 1";
  if (psd && !(t.c1 >= 0.f && t.c2 >= 0.f && t.c3 >= 0.f))
    return "the projected Hessian needs c1, c2 and c3 >= 0 (projection does not commute with a negative weight)";
  return nullptr;
}

}  // namespace

extern "C" {

int tsb_create(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele, const tsb_options_t *opt,
               int device, tsb_handle_t *out) {
  if (!out) return fail<tsb_handle_s>(nullptr, TSB_E_INVALID, "out is null");
  *out = nullptr;
  tsb::PlanConfig pc;
  int nw = 16, ring = 2;
  if (opt) {
    if (opt->warps_per_cta != 0) nw = opt->warps_per_cta;
    if (opt->ring_slots != 0) ring = opt->ring_slots;
    if (opt->tet_cost_x100 > 0) pc.tet_cost = float(opt->tet_cost_x100) / 100.f;
    pc.laplacian_scale = opt->laplacian_scale ? 1 : 0;
    pc.force_global = opt->force_global ? 1 : 0;
    pc.enable_amips = opt->enable_amips ? 1 : 0;
    pc.deterministic = opt->deterministic ? 1 : 0;
  }
  if (nw != 8 && nw != 16) return fail<tsb_handle_s>(nullptr, TSB_E_INVALID, "warps_per_cta must be 8 or 16");
  if (ring < 2 || ring > 8) return fail<tsb_handle_s>(nullptr, TSB_E_INVALID, "ring_slots must be in [2, 8]");
  pc.nw = nw;
  pc.ring_cells = ring * tsb::kCellsPerChunk;   // the requested ring, also when the callback below shrinks it
  const int cpc = tsb::kCellsPerChunk;

  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
    cudaGetLastError();
    return fail<tsb_handle_s>(nullptr, TSB_E_CUDA, "no CUDA device " + std::to_string(device) + " (tssplat_b200 has no CPU path)");
  }
  DeviceGuard guard(device);
  if (!guard.ok) return fail<tsb_handle_s>(nullptr, TSB_E_CUDA, "cannot select CUDA device " + std::to_string(device));
  int sms = 0, smem_optin = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || sms <= 0 ||
      cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess)
    return fail<tsb_handle_s>(nullptr, TSB_E_CUDA, "cannot query the CUDA device");
  pc.area_cap = std::min(tsb::kMaxStagedVerts, std::max(0, (smem_optin - tsb::energy_smem_bytes(nw, 2, cpc, 0, false) - 256) / 32));

  // Called by the plan builder once the component sizes are known: pick the ring size that lets the
  // staging area fit, query occupancy, return the persistent grid.
  int slots = ring, smem = 0, ctas_per_sm = 0;
  pc.grid_cb = [&](int area_verts, bool &global_mode, int &grid, std::string &err) -> int {
    if (!global_mode) {
      int r = ring;
      while (r > 2 && tsb::energy_smem_bytes(nw, r, cpc, area_verts, false) > smem_optin) --r;
      if (tsb::energy_smem_bytes(nw, r, cpc, area_verts, false) > smem_optin) global_mode = true;
      else slots = r;
    }
    if (global_mode) while (slots > 2 && tsb::energy_smem_bytes(nw, slots, cpc, 0, true) > smem_optin) --slots;
    smem = tsb::energy_smem_bytes(nw, slots, cpc, global_mode ? 0 : area_verts, global_mode);
    int ctas = 0;
    cudaError_t e = tsb::energy_occupancy(nw, smem, global_mode, pc.enable_amips != 0, pc.deterministic != 0, &ctas);
    if (e != cudaSuccess || ctas < 1) {
      err = std::string("kernel does not fit the device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "occupancy 0");
      return TSB_E_CUDA;
    }
    ctas_per_sm = std::min(ctas, nw == 16 ? 1 : 2);
    grid = ctas_per_sm * sms;
    return TSB_OK;
  };

  tsb::HostPlan plan;
  std::string err;
  int rc = tsb::build_plan(rest_xyz, tets, n, nele, pc, plan, err);
  if (rc != TSB_OK) return fail<tsb_handle_s>(nullptr, rc, err);

  tsb_handle_t h = new tsb_handle_s();
  h->device = device;
  tsb::KParams &kp = h->kp;
  Rollback<tsb_handle_s> undo(h, tsb_destroy);
  // the plan's tables (at least min_elems elements) and zeroed scratch (at least one element), until one fails
  auto up = [&](const auto &src, auto *&dst, size_t min_elems = 1) {
    if (rc == TSB_OK) rc = device_array(h, dst, min_elems, src.data(), src.size(), false);
  };
  auto zero = [&](size_t elems, auto *&dst) {
    if (rc == TSB_OK) rc = device_array(h, dst, std::max<size_t>(elems, 1));
  };
  up(plan.stream, kp.stream, 16);
  up(plan.X4, kp.X4, 4);
  up(plan.segs, kp.segs);
  up(plan.cta_seg, kp.cta_seg, 2);
  up(plan.wdesc, kp.wdesc, 2);
  up(plan.wseg, kp.wseg, 2);
  up(plan.vlist, kp.vlist);
  up(plan.pos16, kp.pos16, 2);
  up(plan.pos_gid, kp.pos_gid);
  up(plan.orphans, kp.orphans);
  if (pc.enable_amips) {
    up(plan.Bt, kp.Bt, 4);
    up(plan.wtc0, kp.wtc0);
  }
  if (pc.deterministic) {
    // 48 B of corner vectors per tet slot, 8 B of ballot per tet cell, the vertex lists (16 B per tet) and their rows
    const size_t slots = size_t(plan.n_tetcells) * (plan.mode_global ? 32 : 64);
    tsb::DetParams &dp = h->dp;
    if (!pc.enable_amips) up(plan.wtc0, kp.wtc0);
    zero(slots * 3, kp.det_scratch);
    zero(size_t(plan.n_tetcells), kp.det_ballot);
    zero(size_t(plan.n_components), kp.det_flag);
    up(plan.det_rowptr, dp.rowptr);
    up(plan.det_vert, dp.vert);
    up(plan.det_comp_row, dp.comp_row);
    up(plan.det_ent, dp.ent);
    up(plan.det_chunk, dp.chunk, 2);
    dp.scratch = kp.det_scratch;
    dp.ballot = kp.det_ballot;
    dp.flag = kp.det_flag;
    dp.n_chunks = int32_t(plan.det_chunk.size() / 2);
    dp.tpl_log = plan.mode_global ? 0 : 1;
  }
  zero(size_t(plan.n_components), kp.done);
  // per-sphere statistics: 12 B per component of tables, 32 B per (segment, warp) of records
  up(plan.comp_seg, h->sp.comp_seg);
  up(plan.comp_first_vertex, h->sp.comp_first_vertex);
  up(plan.comp_ntets, h->sp.comp_ntets);
  zero(plan.segs.size() * size_t(nw), kp.sph_rec);
  h->sp.rec = kp.sph_rec;
  h->sp.n_components = plan.n_components;
  h->sp.nw = nw;
  up(std::vector<unsigned long long>(size_t(plan.grid) * 4, tsb::kEnergySentinel), kp.cta_energy, 2);
#ifdef TSB_TRACE
  zero(size_t(plan.grid) * tsb::kTraceSlots, kp.trace);
#endif
  if (plan.mode_global) {
    zero(size_t(plan.n), kp.u4g);
    zero(size_t(plan.n), kp.x4g);
  }
  if (rc != TSB_OK) return rc;
  kp.n_orphans = int32_t(plan.orphans.size());
  kp.n_components = plan.n_components;
  kp.n = plan.n;
  kp.vh = plan.vh;
  kp.ring_bytes = tsb::energy_ring_bytes(slots, cpc, plan.mode_global != 0);
  kp.cells_per_chunk = cpc;
  kp.ring_slots = slots;
  kp.stage_bytes = plan.mode_global ? 0 : plan.area_verts * 32;
  h->lc = tsb::LaunchConfig{nw, plan.grid, smem, plan.mode_global, 0, 0, 0};
  h->amips = pc.enable_amips != 0;
  h->det = pc.deterministic != 0;
  h->lap_scale = pc.laplacian_scale;
  h->comp_label = std::move(plan.comp_label);

  tsb_info_t &I = h->info;
  I.n = plan.n; I.nele = plan.nele; I.n_components = plan.n_components; I.grid = plan.grid;
  I.warps_per_cta = nw; I.ctas_per_sm = ctas_per_sm; I.mode_global = plan.mode_global; I.smem_bytes = smem;
  I.ring_slots = slots; I.n_segments = int32_t(plan.segs.size()); I.n_boundary_faces = plan.n_boundary_faces;
  I.max_component_vertices = plan.max_comp_verts; I.nnz = plan.nnz; I.nnz_padded = plan.nnz_padded;
  // bytes one launch requests: the warp streams, rest positions + x per staged component copy, grad
  int64_t staged = 0;
  for (const tsb::SegHdr &s : plan.segs) staged += s.nv;
  I.stream_bytes = int64_t(plan.stream.size()) + (plan.mode_global ? int64_t(plan.n) * (12 + 16 + 64) : staged * (16 + 12 + 2)) +
                   int64_t(plan.n) * 12 + int64_t(plan.segs.size()) * 32 + int64_t(plan.grid) * (16 + 8 * nw);
  undo.commit();
  *out = h;
  return TSB_OK;
}

void tsb_destroy(tsb_handle_t h) {
  if (!h) return;
  DeviceGuard guard(h->device);
  for (int k = 0; k < 2; ++k) {
    if (h->ev_run[k]) cudaEventDestroy(h->ev_run[k]);
    if (h->ev_done[k]) cudaEventDestroy(h->ev_done[k]);
    if (h->s_pipe[k]) cudaStreamDestroy(h->s_pipe[k]);
  }
  for (void *p : h->allocs) cudaFree(p);
  delete h;
}

const char *tsb_last_error(tsb_handle_t h) { return h ? h->err.c_str() : create_err<tsb_handle_s>().c_str(); }

int tsb_get_info(tsb_handle_t h, tsb_info_t *info) {
  if (!h || !info) return TSB_E_INVALID;
  *info = h->info;
  return TSB_OK;
}

static int energy_grad_impl(tsb_handle_t h, const float *x_dev, float c1, float c2, float c3, int32_t order, float gradH,
                            const float *gradH_dev, float *energy_out_dev, int energy4, float *grad_out_dev,
                            tsb_sphere_stats_t *spheres_out_dev, void *stream) {
  if (!h) return TSB_E_INVALID;
  if (!x_dev || !energy_out_dev) return fail(h, TSB_E_INVALID, "x_dev and energy_out_dev must be non-null");
  if (order != 2 && order != 4)
    return fail(h, TSB_E_INVALID, "order must be 2 or 4 (the reference yields zeros for anything else: tet_spheres_cuda.cu:57-63)");
  if (c3 != 0.f && !h->amips) return fail(h, TSB_E_INVALID, "c3 != 0 needs a handle created with tsb_options_t.enable_amips = 1");
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail(h, TSB_E_CUDA, "cannot select the handle's CUDA device");
  tsb::KParams kp = h->kp;
  kp.x = x_dev; kp.grad = grad_out_dev; kp.energy_out = energy_out_dev; kp.gradH_dev = gradH_dev;
  kp.c1 = c1; kp.c2 = c2; kp.c3 = c3; kp.gradH = gradH; kp.order = order; kp.energy4 = energy4;
  tsb::LaunchConfig lc = h->lc;
  lc.amips = c3 != 0.f ? 1 : 0;          // c3 == 0: the very instantiation tsb_energy_grad always ran
  lc.det = h->det && grad_out_dev ? 1 : 0;   // energy only: the default kernel computes the same energies
  lc.sph = spheres_out_dev ? 1 : 0;
  cudaError_t e = tsb::launch_energy_grad(kp, lc, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("energy_grad launch: ") + cudaGetErrorString(e));
  if (lc.det) {
    e = tsb::launch_det_gather(h->dp, grad_out_dev, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("deterministic gather launch: ") + cudaGetErrorString(e));
  }
  if (lc.sph) {
    e = tsb::launch_sphere_fold(h->sp, spheres_out_dev, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("sphere fold launch: ") + cudaGetErrorString(e));
  }
  return TSB_OK;
}

int tsb_energy_grad(tsb_handle_t h, const float *x_dev, float c1, float c2, int32_t order, float gradH,
                    const float *gradH_dev, float *energy_out_dev, float *grad_out_dev, void *stream) {
  return energy_grad_impl(h, x_dev, c1, c2, 0.f, order, gradH, gradH_dev, energy_out_dev, 0, grad_out_dev, nullptr, stream);
}

int tsb_energy_grad_ex(tsb_handle_t h, const float *x_dev, const tsb_terms_t *terms, float gradH, const float *gradH_dev,
                       float *energy_out_dev, float *grad_out_dev, void *stream) {
  if (!h) return TSB_E_INVALID;
  if (!terms) return fail(h, TSB_E_INVALID, "terms is null");
  return energy_grad_impl(h, x_dev, terms->c1, terms->c2, terms->c3, terms->order, gradH, gradH_dev, energy_out_dev, 1, grad_out_dev,
                          nullptr, stream);
}

int tsb_energy_grad_spheres(tsb_handle_t h, const float *x_dev, const tsb_terms_t *terms, float gradH, const float *gradH_dev,
                            float *energy_out_dev, float *grad_out_dev, tsb_sphere_stats_t *spheres_out_dev, void *stream) {
  if (!h) return TSB_E_INVALID;
  if (!terms) return fail(h, TSB_E_INVALID, "terms is null");
  if (!spheres_out_dev) return fail(h, TSB_E_INVALID, "spheres_out_dev must be non-null");
  return energy_grad_impl(h, x_dev, terms->c1, terms->c2, terms->c3, terms->order, gradH, gradH_dev, energy_out_dev, 1, grad_out_dev,
                          spheres_out_dev, stream);
}

static int hvp_impl(tsb_handle_t h, const float *x_dev, const float *v_dev, float c1, float c2, float c3, int32_t order,
                    float gradH, const float *gradH_dev, float *hv_out_dev, float *curv_out_dev, int curv4, void *stream) {
  if (!h) return TSB_E_INVALID;
  if (!x_dev || !v_dev || !hv_out_dev) return fail(h, TSB_E_INVALID, "x_dev, v_dev and hv_out_dev must be non-null");
  if (order != 2 && order != 4) return fail(h, TSB_E_INVALID, "order must be 2 or 4");
  if (c3 != 0.f && !h->amips) return fail(h, TSB_E_INVALID, "c3 != 0 needs a handle created with tsb_options_t.enable_amips = 1");
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail(h, TSB_E_CUDA, "cannot select the handle's CUDA device");
  tsb::KParams kp = h->kp;
  kp.x = x_dev; kp.v = v_dev; kp.grad = hv_out_dev; kp.energy_out = curv_out_dev; kp.gradH_dev = gradH_dev;
  kp.c1 = c1; kp.c2 = c2; kp.c3 = c3; kp.gradH = gradH; kp.order = order; kp.energy4 = curv4;
  tsb::LaunchConfig lc = h->lc;
  lc.amips = c3 != 0.f ? 1 : 0;          // c3 == 0: the very instantiation tsb_hvp runs
  lc.det = h->det ? 1 : 0;
  lc.sph = 0;
  lc.hvp = 1;
  cudaError_t e = tsb::launch_energy_grad(kp, lc, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("hvp launch: ") + cudaGetErrorString(e));
  if (lc.det) {
    e = tsb::launch_det_gather(h->dp, hv_out_dev, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("deterministic gather launch: ") + cudaGetErrorString(e));
  }
  return TSB_OK;
}

int tsb_hvp(tsb_handle_t h, const float *x_dev, const float *v_dev, float c1, float c2, int32_t order, float gradH,
            const float *gradH_dev, float *hv_out_dev, float *curv_out_dev, void *stream) {
  return hvp_impl(h, x_dev, v_dev, c1, c2, 0.f, order, gradH, gradH_dev, hv_out_dev, curv_out_dev, 0, stream);
}

int tsb_hvp_ex(tsb_handle_t h, const float *x_dev, const float *v_dev, const tsb_terms_t *terms, float gradH,
               const float *gradH_dev, float *hv_out_dev, float *curv_out_dev, void *stream) {
  if (!h) return TSB_E_INVALID;
  if (!terms) return fail(h, TSB_E_INVALID, "terms is null");
  return hvp_impl(h, x_dev, v_dev, terms->c1, terms->c2, terms->c3, terms->order, gradH, gradH_dev, hv_out_dev, curv_out_dev,
                  1, stream);
}

int tsb_line_search(tsb_handle_t h, const float *x_dev, const float *d_dev, const tsb_terms_t *terms, const float *alpha_dev,
                    int32_t n_alpha, float *delta_out_dev, float *step_out_dev, float *sphere_delta_out_dev,
                    float *sphere_step_out_dev, void *stream) {
  if (!h) return TSB_E_INVALID;
  if (n_alpha < 1 || n_alpha > TSB_LINE_MAX_ALPHA)
    return fail(h, TSB_E_INVALID, "n_alpha must be in [1, " + std::to_string(TSB_LINE_MAX_ALPHA) + "]");
  if (!terms) return fail(h, TSB_E_INVALID, "terms is null");
  if (!x_dev || !d_dev || !alpha_dev || !delta_out_dev)
    return fail(h, TSB_E_INVALID, "x_dev, d_dev, alpha_dev and delta_out_dev must be non-null");
  if (const char *m = check_terms(h, false, *terms)) return fail(h, TSB_E_INVALID, m);
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail(h, TSB_E_CUDA, "cannot select the handle's CUDA device");
  tsb::KParams kp = h->kp;
  kp.x = x_dev; kp.v = d_dev; kp.grad = nullptr; kp.energy_out = nullptr; kp.gradH_dev = nullptr;
  kp.c1 = terms->c1; kp.c2 = terms->c2; kp.c3 = terms->c3; kp.gradH = 1.f; kp.order = terms->order; kp.energy4 = 0;
  kp.alpha = alpha_dev; kp.n_alpha = n_alpha;
  tsb::LaunchConfig lc = h->lc;
  lc.amips = terms->c3 != 0.f ? 1 : 0;
  lc.det = 0;              // no per-vertex output: the same launch on default and deterministic handles
  lc.sph = 0;
  lc.hvp = 0;
  lc.line = 1;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = tsb::launch_energy_grad(kp, lc, st);
  if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("line search launch: ") + cudaGetErrorString(e));
  e = tsb::launch_line_fold(h->sp, alpha_dev, n_alpha, terms->c1, terms->c2, terms->c3, delta_out_dev, step_out_dev,
                            sphere_delta_out_dev, sphere_step_out_dev, st);
  if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("line search fold launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

int tsb_hess_diag(tsb_handle_t h, const float *x_dev, const tsb_terms_t *terms, float gradH, const float *gradH_dev,
                  float *diag_out_dev, void *stream) {
  if (!h) return TSB_E_INVALID;
  if (!terms) return fail(h, TSB_E_INVALID, "terms is null");
  if (!x_dev || !diag_out_dev) return fail(h, TSB_E_INVALID, "x_dev and diag_out_dev must be non-null");
  if (const char *m = check_terms(h, false, *terms)) return fail(h, TSB_E_INVALID, m);
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail(h, TSB_E_CUDA, "cannot select the handle's CUDA device");
  tsb::KParams kp = h->kp;
  kp.x = x_dev; kp.v = nullptr; kp.grad = diag_out_dev; kp.energy_out = nullptr; kp.gradH_dev = gradH_dev;
  kp.c1 = terms->c1; kp.c2 = terms->c2; kp.c3 = terms->c3; kp.gradH = gradH; kp.order = terms->order; kp.energy4 = 0;
  kp.diag_plane = 0;
  tsb::LaunchConfig lc = h->lc;
  lc.amips = terms->c3 != 0.f ? 1 : 0;
  lc.det = h->det ? 1 : 0;
  lc.sph = 0;
  lc.hvp = 0;
  lc.line = 0;
  lc.diag = 1;
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  // default handle: one launch writes both planes; deterministic handle: a tet slot holds one plane of its corners, so
  // one launch and one gather per plane
  for (int plane = 0; plane < (lc.det ? 2 : 1); ++plane) {
    kp.diag_plane = plane;
    kp.grad = diag_out_dev + size_t(plane) * 3 * size_t(h->info.n);
    cudaError_t e = tsb::launch_energy_grad(kp, lc, st);
    if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("hess_diag launch: ") + cudaGetErrorString(e));
    if (lc.det) {
      e = tsb::launch_det_gather(h->dp, kp.grad, st);
      if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("deterministic gather launch: ") + cudaGetErrorString(e));
    }
  }
  return TSB_OK;
}

/* ---- Newton-CG solve (tsb_solver.cu) ---- */

int tsb_pcg_create(tsb_handle_t h, tsb_pcg_t *out) {
  if (!out) return fail<tsb_pcg_s>(nullptr, TSB_E_INVALID, "out is null");
  *out = nullptr;
  if (!h) return fail<tsb_pcg_s>(nullptr, TSB_E_INVALID, "handle is null");
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail<tsb_pcg_s>(nullptr, TSB_E_CUDA, "cannot select the handle's CUDA device");
  tsb::PcgLists L;
  tsb::build_pcg_lists(h->comp_label, h->info.n_components, L);
  tsb_pcg_t s = new tsb_pcg_s();
  s->h = h;
  s->device = h->device;
  tsb::PcgParams &P = s->P;
  const size_t n = size_t(h->info.n), n3 = 3 * n;
  Rollback<tsb_pcg_s> undo(s, tsb_pcg_destroy);
  int rc = device_array(s, P.vert, 0, L.vert.data(), L.vert.size());
  if (rc == TSB_OK) rc = device_array(s, P.comp_chunk, 0, L.comp_chunk.data(), L.comp_chunk.size());
  if (rc == TSB_OK) rc = device_array(s, P.chunk, 0, L.chunk.data(), L.chunk.size());
  if (rc == TSB_OK) rc = device_array(s, P.r, n3);
  if (rc == TSB_OK) rc = device_array(s, P.z, n3);
  if (rc == TSB_OK) rc = device_array(s, P.p, n3);     // zero on vertices no tet references, and stays so
  if (rc == TSB_OK) rc = device_array(s, P.Hp, n3);
  if (rc == TSB_OK) rc = device_array(s, P.pinv, 2 * n3);
  if (rc == TSB_OK) rc = device_array(s, P.part, 3 * (L.chunk.size() / 3));
  if (rc == TSB_OK) rc = device_array(s, P.comp, size_t(h->info.n_components));
  if (rc == TSB_OK) rc = device_array(s, P.active, 1);
  if (rc != TSB_OK) return rc;
  P.orphans = h->kp.orphans; P.n_orphans = h->kp.n_orphans;
  P.n_chunks = int32_t(L.chunk.size() / 3); P.n_components = h->info.n_components; P.n = h->info.n;
  cudaError_t e = cudaMallocHost(reinterpret_cast<void **>(&s->active_host), sizeof(int32_t));
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->ev, cudaEventDisableTiming);
  if (e == cudaSuccess) e = tsb::launch_pcg_blocks(P, nullptr, 0.f, nullptr, nullptr);     // identity preconditioner
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("tsb_pcg_create: ") + cudaGetErrorString(e));
  undo.commit();
  *out = s;
  return TSB_OK;
}

void tsb_pcg_destroy(tsb_pcg_t s) {
  if (!s) return;
  DeviceGuard guard(s->device);
  if (s->ev) cudaEventDestroy(s->ev);
  if (s->active_host) cudaFreeHost(s->active_host);
  for (void *p : s->allocs) cudaFree(p);
  delete s;
}

const char *tsb_pcg_last_error(tsb_pcg_t s) { return s ? s->err.c_str() : create_err<tsb_pcg_s>().c_str(); }

int64_t tsb_pcg_device_bytes(tsb_pcg_t s) { return s ? s->device_bytes : 0; }

int tsb_pcg_set_blocks(tsb_pcg_t s, const float *diag_dev, float rel_floor, float *inv_out_dev, void *stream) {
  return tsb_pcg_set_blocks_ex(s, diag_dev, rel_floor, nullptr, inv_out_dev, stream);
}

int tsb_pcg_set_blocks_ex(tsb_pcg_t s, const float *diag_dev, float rel_floor, const float *shift_dev, float *inv_out_dev,
                          void *stream) {
  if (!s) return TSB_E_INVALID;
  if (!(rel_floor >= 0.f)) return fail(s, TSB_E_INVALID, "rel_floor must be >= 0");
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = diag_dev && shift_dev ? tsb::launch_pcg_blocks_shift(s->P, diag_dev, rel_floor, shift_dev, inv_out_dev, st)
                                        : tsb::launch_pcg_blocks(s->P, diag_dev, rel_floor, inv_out_dev, st);
  if (e == cudaSuccess && s->coarse) e = tsb::launch_coarse_factor(s->P, s->co, diag_dev ? shift_dev : nullptr, nullptr, st);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("preconditioner launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

}  // extern "C"

namespace {

// hv = c1 M v (the exact product with c2 = c3 = 0: its tet pass adds exact zeros) + c2 P(H_b) v + c3 P(H_a) v at the
// workspace's last projection; curv (optional, device float[4]) as tsb_pcg_hvp_psd reports it
int psd_product(tsb_pcg_t s, const float *x_dev, const float *v_dev, const tsb_terms_t &t, float *hv, float *curv,
                cudaStream_t st) {
  const int rc = hvp_impl(s->h, x_dev, v_dev, t.c1, 0.f, 0.f, t.order, 1.f, nullptr, hv, curv ? s->Q.curv_m : nullptr, 1, st);
  if (rc != TSB_OK) return fail(s, rc, s->h->err);
  cudaError_t e = tsb::launch_psd_apply(s->Q, v_dev, t.c2, t.c3, curv != nullptr, hv, st);
  if (e == cudaSuccess && curv) e = tsb::launch_psd_curv(s->Q, t.c1, t.c2, t.c3, curv, st);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("projected product launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

int psd_project(tsb_pcg_t s, const float *x_dev, const tsb_terms_t &t, cudaStream_t st) {
  const cudaError_t e = tsb::launch_psd_project(s->Q, x_dev, t.order, t.c3 != 0.f ? 1 : 0, st);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("projection launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

// The coarse matrix's partials at x (PSD mode: after the solve's projection launch, so the same x gives the same
// operator bits) and, with factor, its unshifted E+.  A Newton step leaves the factorisation to tsb_pcg_set_blocks_ex,
// which follows with the step's shift.
int coarse_form(tsb_pcg_t s, const float *x_dev, const tsb_terms_t &t, bool factor, cudaStream_t st) {
  if (s->psd) {
    const int rc = psd_project(s, x_dev, t, st);
    if (rc != TSB_OK) return rc;
  }
  cudaError_t e = tsb::launch_coarse_tets(s->co, x_dev, t.order, t.c2, t.c3, s->psd ? &s->Q : nullptr, st);
  if (e == cudaSuccess && factor) e = tsb::launch_coarse_factor(s->P, s->co, nullptr, nullptr, st);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("coarse launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

}  // namespace

extern "C" {

int tsb_pcg_enable_psd(tsb_pcg_t s, const float *rest_xyz, const int32_t *tets, int32_t nele) {
  if (!s) return TSB_E_INVALID;
  if (s->psd) return fail(s, TSB_E_INVALID, "the projected Hessian is already enabled on this workspace");
  if (!rest_xyz || !tets) return fail(s, TSB_E_INVALID, "rest_xyz and tets must be non-null");
  const tsb_handle_t h = s->h;
  if (nele != h->info.nele)
    return fail(s, TSB_E_INVALID, "nele = " + std::to_string(nele) + " but the handle has " + std::to_string(h->info.nele) + " tets");
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  int rc = refuse_capture(s, cudaStreamLegacy, "tsb_pcg_enable_psd allocates device memory and cannot run while a stream is being captured");
  if (rc != TSB_OK) return rc;
  const int32_t n = h->info.n;
  const size_t ne = size_t(nele);
  // the mesh: every vertex in range, every tet inside one component, B = Dm^-1 in fp64 stored as fp32
  tsb::TetTables T;
  std::string err;
  rc = tsb::build_tet_tables(rest_xyz, tets, n, nele, &h->comp_label, T, err);
  if (rc != TSB_OK) return fail(s, rc, err);
  tsb::PsdParams Q{};
  Q.nele = nele; Q.n = n; Q.n_blocks = int32_t((ne + tsb::kPsdT - 1) / tsb::kPsdT);
  Rollback<tsb_pcg_s> undo(s);
  rc = device_array(s, Q.tets, 0, T.tets.data(), T.tets.size());
  if (rc == TSB_OK) rc = device_array(s, Q.B, 0, T.B.data(), T.B.size());
  if (rc == TSB_OK) rc = device_array(s, Q.op, tsb::kPsdOpFloats * ne);
  if (rc == TSB_OK) rc = device_array(s, Q.kind, ne);
  if (rc == TSB_OK) rc = device_array(s, Q.corner, 12 * ne);
  if (rc == TSB_OK) rc = device_array(s, Q.inc_ptr, 0, T.inc_ptr.data(), T.inc_ptr.size());
  if (rc == TSB_OK) rc = device_array(s, Q.inc, 0, T.inc.data(), T.inc.size());
  if (rc == TSB_OK) rc = device_array(s, Q.part, 2 * size_t(Q.n_blocks));
  if (rc == TSB_OK) rc = device_array(s, Q.curv_m, 4);
  if (rc != TSB_OK) return rc;       // the rollback leaves the workspace as it was
  undo.commit();
  s->Q = Q;
  s->psd = true;
  return TSB_OK;
}

int tsb_pcg_hvp_psd(tsb_pcg_t s, const float *x_dev, const float *v_dev, const tsb_terms_t *terms, float *hv_out_dev,
                    float *curv_out_dev, void *stream) {
  if (!s) return TSB_E_INVALID;
  if (!s->psd) return fail(s, TSB_E_INVALID, "tsb_pcg_hvp_psd needs a workspace after tsb_pcg_enable_psd");
  if (!x_dev || !v_dev || !terms || !hv_out_dev) return fail(s, TSB_E_INVALID, "x_dev, v_dev, terms and hv_out_dev must be non-null");
  if (hv_out_dev == v_dev || hv_out_dev == x_dev)
    return fail(s, TSB_E_INVALID, "hv_out_dev must not be x_dev or v_dev: hv is written before v and x are read for the last time");
  if (const char *m = check_terms(s->h, true, *terms)) return fail(s, TSB_E_INVALID, m);
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc = psd_project(s, x_dev, *terms, st);
  if (rc == TSB_OK) rc = psd_product(s, x_dev, v_dev, *terms, hv_out_dev, curv_out_dev, st);
  return rc;
}

int tsb_pcg_solve(tsb_pcg_t s, const float *x_dev, const float *b_dev, const tsb_terms_t *terms, const tsb_pcg_options_t *opt,
                  float *d_out_dev, tsb_pcg_sphere_t *spheres_out_dev, int32_t *iters_run_out, void *stream) {
  return tsb_pcg_solve_ex(s, x_dev, b_dev, terms, opt, nullptr, d_out_dev, spheres_out_dev, iters_run_out, stream);
}

}  // extern "C"

namespace {

// tsb_pcg_solve_ex, and tsb_pcg_solve_tr when radius_dev != nullptr
int pcg_solve_impl(tsb_pcg_t s, const float *x_dev, const float *b_dev, const tsb_terms_t *terms, const tsb_pcg_options_t *opt,
                   const float *shift_dev, const float *radius_dev, float *d_out_dev, tsb_pcg_sphere_t *spheres_out_dev,
                   int32_t *iters_run_out, void *stream) {
  if (!x_dev || !b_dev || !d_out_dev || !terms || !opt)
    return fail(s, TSB_E_INVALID, "x_dev, b_dev, d_out_dev, terms and opt must be non-null");
  if (opt->max_iter < 1) return fail(s, TSB_E_INVALID, "max_iter must be >= 1");
  if (!(opt->rtol >= 0.f)) return fail(s, TSB_E_INVALID, "rtol must be >= 0");
  if (opt->check_every < 0) return fail(s, TSB_E_INVALID, "check_every must be >= 0");
  if (const char *m = check_terms(s->h, s->psd, *terms)) return fail(s, TSB_E_INVALID, m);
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (opt->check_every > 0) {          // the termination check waits on the host: not possible inside a stream capture
    const int rc = refuse_capture(s, st, "check_every > 0 reads the host and cannot be captured in a CUDA graph: use check_every = 0");
    if (rc != TSB_OK) return rc;
  }
  if (radius_dev) {     // the recurrence state: the dir kernel of iteration 0 writes it before any kernel reads it
    const int rc = alloc_once(s, size_t(s->P.n_components), &s->tr, st,
                              "the first tsb_pcg_solve_tr of a workspace allocates device memory and cannot be captured in a "
                              "CUDA graph: make one call outside any capture first");
    if (rc != TSB_OK) return rc;
  }
  const tsb::TrParams tp{radius_dev, s->tr};
  const tsb::TrParams *tr = radius_dev ? &tp : nullptr;
  const tsb::PcgParams &P = s->P;
  if (s->psd) {                        // x does not change during the solve: one projection
    const int rc = psd_project(s, x_dev, *terms, st);
    if (rc != TSB_OK) return rc;
  }
  const tsb::SgsParams *sgs = s->sgs ? &s->G : nullptr;
  const tsb::CoarseParams *co = s->coarse ? &s->co : nullptr;
  cudaError_t e = tsb::launch_pcg_begin(P, b_dev, d_out_dev, tr, st, sgs, co);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("solver launch: ") + cudaGetErrorString(e));
  int32_t it = 0;
  while (it < opt->max_iter) {
    if (s->psd) {
      const int rc = psd_product(s, x_dev, P.p, *terms, P.Hp, nullptr, st);
      if (rc != TSB_OK) return rc;
    } else {
      const int rc = hvp_impl(s->h, x_dev, P.p, terms->c1, terms->c2, terms->c3, terms->order, 1.f, nullptr, P.Hp, nullptr, 1, st);
      if (rc != TSB_OK) return fail(s, rc, s->h->err);
    }
    e = tsb::launch_pcg_step(P, d_out_dev, it, opt->rtol, shift_dev, tr, st, sgs, co);
    if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("solver launch: ") + cudaGetErrorString(e));
    ++it;
    if (opt->check_every > 0 && it % opt->check_every == 0 && it < opt->max_iter) {
      e = tsb::launch_pcg_count(P, st);
      if (e == cudaSuccess) e = cudaMemcpyAsync(s->active_host, P.active, sizeof(int32_t), cudaMemcpyDeviceToHost, st);
      if (e == cudaSuccess) e = cudaEventRecord(s->ev, st);
      if (e == cudaSuccess) e = cudaEventSynchronize(s->ev);
      if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("solver termination check: ") + cudaGetErrorString(e));
      if (*s->active_host == 0) break;
    }
  }
  if (iters_run_out) *iters_run_out = it;
  if (spheres_out_dev) {
    e = tsb::launch_pcg_records(P, b_dev, d_out_dev, spheres_out_dev, st);
    if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("solver record launch: ") + cudaGetErrorString(e));
  }
  return TSB_OK;
}

}  // namespace

extern "C" {

int tsb_pcg_solve_ex(tsb_pcg_t s, const float *x_dev, const float *b_dev, const tsb_terms_t *terms, const tsb_pcg_options_t *opt,
                     const float *shift_dev, float *d_out_dev, tsb_pcg_sphere_t *spheres_out_dev, int32_t *iters_run_out,
                     void *stream) {
  if (!s) return TSB_E_INVALID;
  return pcg_solve_impl(s, x_dev, b_dev, terms, opt, shift_dev, nullptr, d_out_dev, spheres_out_dev, iters_run_out, stream);
}

int tsb_pcg_solve_tr(tsb_pcg_t s, const float *x_dev, const float *b_dev, const tsb_terms_t *terms, const tsb_pcg_options_t *opt,
                     const float *shift_dev, const float *radius_dev, float *d_out_dev, tsb_pcg_sphere_t *spheres_out_dev,
                     int32_t *iters_run_out, void *stream) {
  if (!s) return TSB_E_INVALID;
  if (!radius_dev) return fail(s, TSB_E_INVALID, "radius_dev must be non-null");
  return pcg_solve_impl(s, x_dev, b_dev, terms, opt, shift_dev, radius_dev, d_out_dev, spheres_out_dev, iters_run_out, stream);
}

int tsb_sphere_axpy(tsb_pcg_t s, const float *x_dev, const float *a_sphere_dev, const float *d_dev, float *out_dev,
                    void *stream) {
  if (!s) return TSB_E_INVALID;
  if (!x_dev || !a_sphere_dev || !d_dev || !out_dev)
    return fail(s, TSB_E_INVALID, "x_dev, a_sphere_dev, d_dev and out_dev must be non-null");
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaError_t e = tsb::launch_sphere_axpy(s->P, x_dev, a_sphere_dev, d_dev, out_dev, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("sphere axpy launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

/* ---- Damped Newton step (tsb_solver.cu) ---- */

int tsb_newton_create(tsb_pcg_t s, tsb_newton_t *out) {
  if (!out) return fail<tsb_newton_s>(nullptr, TSB_E_INVALID, "out is null");
  *out = nullptr;
  if (!s) return fail<tsb_newton_s>(nullptr, TSB_E_INVALID, "solver workspace is null");
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail<tsb_newton_s>(nullptr, TSB_E_CUDA, "cannot select the handle's CUDA device");
  tsb_newton_t nw = new tsb_newton_s();
  nw->s = s;
  nw->device = s->h->device;
  tsb::NewtonParams &W = nw->W;
  const size_t n3 = 3 * size_t(s->P.n), S = size_t(s->P.n_components), K = TSB_LINE_MAX_ALPHA;
  std::vector<float> alphas(K);
  for (size_t k = 0; k < K; ++k) alphas[k] = std::ldexp(1.f, -int(k));
  Rollback<tsb_newton_s> undo(nw, tsb_newton_destroy);
  int rc = device_array(nw, W.b, n3);
  if (rc == TSB_OK) rc = device_array(nw, W.d, n3);
  if (rc == TSB_OK) rc = device_array(nw, W.diag, 2 * n3);
  if (rc == TSB_OK) rc = device_array(nw, W.shift, S);
  if (rc == TSB_OK) rc = device_array(nw, W.alpha_sphere, S);
  if (rc == TSB_OK) rc = device_array(nw, W.alphas, 0, alphas.data(), K);
  if (rc == TSB_OK) rc = device_array(nw, W.sphere_delta, S * K * 4);
  if (rc == TSB_OK) rc = device_array(nw, W.sphere_step, S);
  if (rc == TSB_OK) rc = device_array(nw, W.part, 3 * size_t(s->P.n_chunks));
  if (rc == TSB_OK) rc = device_array(nw, W.comp, S);     // zero: ACTIVE, mu not initialised
  if (rc == TSB_OK) rc = device_array(nw, nw->energy, 4);
  if (rc == TSB_OK) rc = device_array(nw, nw->delta, K * 4);
  if (rc != TSB_OK) return rc;
  undo.commit();
  *out = nw;
  return TSB_OK;
}

void tsb_newton_destroy(tsb_newton_t nw) {
  if (!nw) return;
  DeviceGuard guard(nw->device);
  for (void *p : nw->allocs) cudaFree(p);
  delete nw;
}

const char *tsb_newton_last_error(tsb_newton_t nw) { return nw ? nw->err.c_str() : create_err<tsb_newton_s>().c_str(); }

int64_t tsb_newton_device_bytes(tsb_newton_t nw) { return nw ? nw->device_bytes : 0; }

int tsb_newton_reset(tsb_newton_t nw, void *stream) {
  if (!nw) return TSB_E_INVALID;
  DeviceGuard guard(nw->s->h->device);
  if (!guard.ok) return fail(nw, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const size_t S = size_t(nw->s->P.n_components);
  cudaError_t e = cudaMemsetAsync(nw->W.comp, 0, S * sizeof(tsb::NewtonComp), static_cast<cudaStream_t>(stream));
  if (e == cudaSuccess && nw->tr_state) e = cudaMemsetAsync(nw->tr_state, 0, S * sizeof(tsb::TrState), static_cast<cudaStream_t>(stream));
  if (e == cudaSuccess && nw->lb.comp) e = cudaMemsetAsync(nw->lb.comp, 0, S * sizeof(tsb::LbfgsComp), static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(nw, TSB_E_CUDA, std::string("reset: ") + cudaGetErrorString(e));
  return TSB_OK;
}

}  // extern "C"

namespace {

// The options a kind of Newton step adds to those every step has: "" when they hold, or the message of the first broken
std::string rule_error(const tsb_newton_options_t &o) {
  if (!(o.tau > 0.f) || !std::isfinite(o.tau)) return "tau must be finite and > 0";
  if (!(o.mu_min > 0.f) || !(o.mu_min <= o.mu_max) || !std::isfinite(o.mu_max))
    return "mu_min and mu_max must satisfy 0 < mu_min <= mu_max < inf";
  if (!(o.sigma > 0.f && o.sigma < 1.f)) return "sigma must be in (0, 1)";
  if (o.n_alpha < 1 || o.n_alpha > TSB_LINE_MAX_ALPHA) return "n_alpha must be in [1, " + std::to_string(TSB_LINE_MAX_ALPHA) + "]";
  return "";
}

std::string rule_error(const tsb_newton_tr_options_t &o) {
  if (!(o.radius_init > 0.f) || !std::isfinite(o.radius_init)) return "radius_init must be finite and > 0";
  if (!(o.radius_min > 0.f) || !(o.radius_min <= o.radius_max) || !std::isfinite(o.radius_max))
    return "radius_min and radius_max must satisfy 0 < radius_min <= radius_max < inf";
  if (!(o.accept >= 0.f && o.accept < 0.25f)) return "accept must be in [0, 1/4)";
  return "";
}

// The pointer rules of every Newton step: x, terms and opt set, the proximal pair (anchor_dev and weight_dev both null:
// objective E, or both set, the anchor not x).
int newton_pointers_check(tsb_newton_t nw, const float *x_dev, const float *anchor_dev, const float *weight_dev,
                          const tsb_terms_t *terms, const void *opt) {
  if (!x_dev || !terms || !opt) return fail(nw, TSB_E_INVALID, "x_dev, terms and opt must be non-null");
  if (!anchor_dev != !weight_dev)
    return fail(nw, TSB_E_INVALID, "anchor_dev and weight_dev must be both null (objective E) or both set (proximal objective)");
  if (anchor_dev && anchor_dev == x_dev)
    return fail(nw, TSB_E_INVALID, "anchor_dev must not be x_dev: x is updated in place while the anchor is read");
  return TSB_OK;
}

// The argument rules of every Newton step: the pointers, the options all steps have, those of the step's kind (O), and
// the terms.
template <class O>
int newton_check(tsb_newton_t nw, const float *x_dev, const float *anchor_dev, const float *weight_dev, const tsb_terms_t *terms,
                 const O *opt) {
  const int rc = newton_pointers_check(nw, x_dev, anchor_dev, weight_dev, terms, opt);
  if (rc != TSB_OK) return rc;
  const O &o = *opt;
  if (o.max_iter < 1) return fail(nw, TSB_E_INVALID, "max_iter must be >= 1");
  if (!(o.rtol >= 0.f)) return fail(nw, TSB_E_INVALID, "rtol must be >= 0");
  if (!(o.rel_floor >= 0.f)) return fail(nw, TSB_E_INVALID, "rel_floor must be >= 0");
  if (!(o.gtol >= 0.f)) return fail(nw, TSB_E_INVALID, "gtol must be >= 0");
  if (!(o.eta > 0.f && o.eta <= 1.f)) return fail(nw, TSB_E_INVALID, "eta must be in (0, 1]");
  for (int32_t r : o.reserved)
    if (r != 0) return fail(nw, TSB_E_INVALID, "reserved fields must be 0");
  const std::string rule = rule_error(o);
  if (!rule.empty()) return fail(nw, TSB_E_INVALID, rule);
  if (const char *m = check_terms(nw->s->h, nw->s->psd, *terms)) return fail(nw, TSB_E_INVALID, m);
  return TSB_OK;
}

// What tells the Newton steps apart.  The damped step (tsb_newton_step, tsb_newton_prox_step) solves with the shift mu_c
// (+ w_c) and no radius, line-searches n_alpha step sizes and decides by the damping rule; the trust-region step
// (tsb_newton_tr_step, _ex) solves with the shift w_c of a proximal step (none otherwise) inside the radius, line-searches
// alpha = 1 (with backtracking: bt.n_alpha step sizes) and decides by the trust-region rule.
struct NewtonStep {
  bool damped;
  tsb::NewtonRule lm{};
  tsb_newton_sphere_t *lm_out = nullptr;
  tsb::NewtonTrRule tr{};
  bool backtrack = false;
  tsb::NewtonBacktrack bt{};
  tsb_newton_tr_sphere_t *tr_out = nullptr;
  tsb_pcg_options_t po;
  float rel_floor;
  int32_t n_alpha;

  NewtonStep(const tsb_newton_options_t &o, tsb_newton_sphere_t *out)
      : damped(true), lm{o.tau, o.mu_min, o.mu_max, o.gtol, o.sigma, o.eta, o.n_alpha}, lm_out(out),
        po{o.max_iter, o.rtol, 0, {0, 0, 0, 0, 0}}, rel_floor(o.rel_floor), n_alpha(o.n_alpha) {}
  NewtonStep(const tsb_newton_tr_options_t &o, const tsb_newton_backtrack_t *b, tsb_newton_tr_sphere_t *out)
      : damped(false), tr{o.gtol, o.radius_init, o.radius_min, o.radius_max, o.accept, o.eta}, backtrack(b != nullptr),
        bt{b ? b->sigma : 0.f, b ? b->n_alpha : 1}, tr_out(out), po{o.max_iter, o.rtol, 0, {0, 0, 0, 0, 0}},
        rel_floor(o.rel_floor), n_alpha(b ? b->n_alpha : 1) {}
};

// The first phases of every Newton step: b = -grad at x, the diagonal blocks (from the assembled matrix on an SGS
// workspace), E_c on a coarse workspace, then the prep kernel: b_c = 0 on frozen spheres (prox: b -= w (x - y)).
int newton_rhs(tsb_newton_t nw, const float *x_dev, const tsb_terms_t *terms, const tsb::ProxParams *prox, cudaStream_t st) {
  tsb_pcg_t s = nw->s;
  tsb_handle_t h = s->h;
  const tsb::NewtonParams &W = nw->W;
  int rc = energy_grad_impl(h, x_dev, terms->c1, terms->c2, terms->c3, terms->order, -1.f, nullptr, nw->energy, 1, W.b, nullptr, st);
  if (rc != TSB_OK) return fail(nw, rc, h->err);
  if (s->sgs) {         // the diagonal blocks of the matrix the sweep uses
    rc = tsb_pcg_set_matrix(s, x_dev, terms, W.diag, st);
    if (rc != TSB_OK) return fail(nw, rc, s->err);
  } else {
    rc = tsb_hess_diag(h, x_dev, terms, 1.f, nullptr, W.diag, st);
    if (rc != TSB_OK) return fail(nw, rc, h->err);
  }
  if (s->coarse) {      // E_c at x; the step's tsb_pcg_set_blocks_ex factors it with the step's shift
    rc = coarse_form(s, x_dev, *terms, false, st);
    if (rc != TSB_OK) return fail(nw, rc, s->err);
  }
  const cudaError_t e = tsb::launch_newton_prep(s->P, W, prox, st);
  if (e != cudaSuccess) return fail(nw, TSB_E_CUDA, std::string("newton launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

// One Newton step of every sphere after its arguments are checked: the first call's allocations, then gradient, diagonal
// blocks, prep (damped: and the shift), preconditioner, (trust region: the radius), solve, dots, line search, decision and
// the step itself.
int newton_run(tsb_newton_t nw, float *x_dev, const float *anchor_dev, const float *weight_dev, const tsb_terms_t *terms,
               const NewtonStep &k, void *stream) {
  tsb_pcg_t s = nw->s;
  tsb_handle_t h = s->h;
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail(nw, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const char *refusal = k.damped ? "the first tsb_newton_prox_step of a workspace allocates device memory and cannot be "
                                   "captured in a CUDA graph: make one call outside any capture first"
                                 : "the first tsb_newton_tr_step of a workspace (and the first proximal one) allocates device memory "
                                   "and cannot be captured in a CUDA graph: make one call outside any capture first";
  const size_t S = size_t(s->P.n_components);
  int rc = TSB_OK;
  if (!k.damped) {      // the radius state (every radius to be initialised) and its fp32 radius
    rc = alloc_once(nw, S, &nw->tr_state, st, refusal, true);
    if (rc == TSB_OK) rc = alloc_once(nw, S, &nw->tr_radius, st, refusal);
  }
  // the d.(x - y) partials, never read before written
  if (rc == TSB_OK && anchor_dev) rc = alloc_once(nw, size_t(s->P.n_chunks), &nw->prox_part, st, refusal);
  if (rc != TSB_OK) return rc;
  if (!k.damped) {      // the solve's recurrence state, as a first tsb_pcg_solve_tr allocates it
    rc = alloc_once(s, S, &s->tr, st, refusal);
    if (rc != TSB_OK) return fail(nw, rc, s->err);
  }
  const tsb::NewtonParams &W = nw->W;
  const tsb::ProxParams pp{x_dev, anchor_dev, weight_dev, nw->prox_part};
  const tsb::ProxParams *prox = anchor_dev ? &pp : nullptr;
  const tsb::NewtonTrParams T{nw->tr_state, nw->tr_radius, s->tr};
  // the trust-region step's shift w_c: an unusable w_c only reaches a sphere whose b_c is 0
  const float *shift = k.damped ? W.shift : weight_dev;
  // b = -grad, the diagonal blocks; frozen spheres' b = 0 (prox: b -= w (x - y)); damped: mu on a first step
  rc = newton_rhs(nw, x_dev, terms, prox, st);
  if (rc != TSB_OK) return rc;
  cudaError_t e = cudaSuccess;
  if (k.damped) e = tsb::launch_newton_shift(s->P, W, k.lm, prox, st);
  if (e != cudaSuccess) return fail(nw, TSB_E_CUDA, std::string("newton launch: ") + cudaGetErrorString(e));
  // the preconditioner; trust region: the radius on a first step
  rc = tsb_pcg_set_blocks_ex(s, W.diag, k.rel_floor, shift, nullptr, st);
  if (rc != TSB_OK) return fail(nw, rc, s->err);
  if (!k.damped) {
    e = tsb::launch_newton_tr_radius(s->P, W, T, k.tr, st, s->sgs ? &s->G : nullptr);
    if (e != cudaSuccess) return fail(nw, TSB_E_CUDA, std::string("newton launch: ") + cudaGetErrorString(e));
  }
  // the solve
  rc = pcg_solve_impl(s, x_dev, W.b, terms, &k.po, shift, k.damped ? nullptr : nw->tr_radius, W.d, nullptr, nullptr, st);
  if (rc != TSB_OK) return fail(nw, rc, s->err);
  // b.d and |d|^2 (prox: and d.(x - y)) per chunk; the line search at 2^-k, k < n_alpha, per sphere
  e = tsb::launch_newton_dots(s->P, W, prox, st);
  if (e != cudaSuccess) return fail(nw, TSB_E_CUDA, std::string("newton launch: ") + cudaGetErrorString(e));
  rc = tsb_line_search(h, x_dev, W.d, terms, W.alphas, k.n_alpha, nw->delta, nullptr, W.sphere_delta, W.sphere_step, st);
  if (rc != TSB_OK) return fail(nw, rc, h->err);
  // decision, step
  e = k.damped ? tsb::launch_newton_decide(s->P, W, k.lm, prox, k.lm_out, st)
               : tsb::launch_newton_tr_decide(s->P, W, T, k.tr, prox, k.backtrack ? &k.bt : nullptr, k.tr_out, st);
  if (e == cudaSuccess) e = tsb::launch_sphere_axpy(s->P, x_dev, W.alpha_sphere, W.d, x_dev, st);
  if (e != cudaSuccess) return fail(nw, TSB_E_CUDA, std::string("newton launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

}  // namespace

extern "C" {

int tsb_newton_step(tsb_newton_t nw, float *x_dev, const tsb_terms_t *terms, const tsb_newton_options_t *opt,
                    tsb_newton_sphere_t *records_out_dev, void *stream) {
  if (!nw) return TSB_E_INVALID;
  const int rc = newton_check(nw, x_dev, nullptr, nullptr, terms, opt);
  if (rc != TSB_OK) return rc;
  return newton_run(nw, x_dev, nullptr, nullptr, terms, NewtonStep(*opt, records_out_dev), stream);
}

int tsb_newton_prox_step(tsb_newton_t nw, float *x_dev, const float *anchor_dev, const float *weight_dev,
                         const tsb_terms_t *terms, const tsb_newton_options_t *opt, tsb_newton_sphere_t *records_out_dev,
                         void *stream) {
  if (!nw) return TSB_E_INVALID;
  if (!anchor_dev || !weight_dev) return fail(nw, TSB_E_INVALID, "anchor_dev and weight_dev must be non-null");
  const int rc = newton_check(nw, x_dev, anchor_dev, weight_dev, terms, opt);
  if (rc != TSB_OK) return rc;
  return newton_run(nw, x_dev, anchor_dev, weight_dev, terms, NewtonStep(*opt, records_out_dev), stream);
}

int tsb_newton_tr_step(tsb_newton_t nw, float *x_dev, const float *anchor_dev, const float *weight_dev, const tsb_terms_t *terms,
                       const tsb_newton_tr_options_t *opt, tsb_newton_tr_sphere_t *records_out_dev, void *stream) {
  return tsb_newton_tr_step_ex(nw, x_dev, anchor_dev, weight_dev, terms, opt, nullptr, records_out_dev, stream);
}

int tsb_newton_tr_step_ex(tsb_newton_t nw, float *x_dev, const float *anchor_dev, const float *weight_dev, const tsb_terms_t *terms,
                          const tsb_newton_tr_options_t *opt, const tsb_newton_backtrack_t *bt,
                          tsb_newton_tr_sphere_t *records_out_dev, void *stream) {
  if (!nw) return TSB_E_INVALID;
  const int rc = newton_check(nw, x_dev, anchor_dev, weight_dev, terms, opt);
  if (rc != TSB_OK) return rc;
  if (nw->s->coarse)    // the two-level norm is near-singular along the coarse modes: the radius then admits long affine
                        // moves the gain ratio rejects, and the steps stall (DESIGN.md section 5, "Affine coarse space")
    return fail(nw, TSB_E_INVALID, "the trust-region steps do not take a workspace with the coarse space (tsb_pcg_enable_coarse)");
  if (bt) {
    if (bt->n_alpha < 2 || bt->n_alpha > TSB_LINE_MAX_ALPHA)
      return fail(nw, TSB_E_INVALID, "n_alpha must be in [2, " + std::to_string(TSB_LINE_MAX_ALPHA) + "]");
    if (!(bt->sigma > 0.f && bt->sigma < 0.5f)) return fail(nw, TSB_E_INVALID, "sigma must be in (0, 1/2)");
    for (int32_t r : bt->reserved)
      if (r != 0) return fail(nw, TSB_E_INVALID, "reserved fields must be 0");
  }
  return newton_run(nw, x_dev, anchor_dev, weight_dev, terms, NewtonStep(*opt, bt, records_out_dev), stream);
}

}  // extern "C"

namespace {

// The L-BFGS options: "" when they hold, or the message of the first broken
std::string lbfgs_rule_error(const tsb_newton_lbfgs_options_t &o) {
  if (o.m < 1 || o.m > TSB_LBFGS_MAX_M) return "m must be in [1, " + std::to_string(TSB_LBFGS_MAX_M) + "]";
  if (!(o.gtol >= 0.f)) return "gtol must be >= 0";
  if (!(o.sigma > 0.f && o.sigma < 1.f)) return "sigma must be in (0, 1)";
  if (!(o.eta > 0.f && o.eta <= 1.f)) return "eta must be in (0, 1]";
  if (o.n_alpha < 1 || o.n_alpha > TSB_LINE_MAX_ALPHA) return "n_alpha must be in [1, " + std::to_string(TSB_LINE_MAX_ALPHA) + "]";
  if (!(o.rel_floor >= 0.f)) return "rel_floor must be >= 0";
  if (!(o.curv_eps >= 0.f) || !std::isfinite(o.curv_eps)) return "curv_eps must be finite and >= 0";
  for (int32_t r : o.reserved)
    if (r != 0) return "reserved fields must be 0";
  return "";
}

// The L-BFGS state of a workspace, allocated by its first L-BFGS step (every history empty, no sphere moved).
int lbfgs_alloc(tsb_newton_t nw, int32_t m, cudaStream_t st) {
  if (nw->lb.m) return TSB_OK;
  const char *refusal = "the first tsb_newton_lbfgs_step of a workspace allocates device memory and cannot be captured in a "
                        "CUDA graph: make one call outside any capture first";
  const tsb::PcgParams &P = nw->s->P;
  const size_t rows = size_t(P.n - P.n_orphans), S = size_t(P.n_components), M1 = size_t(m) + 1;
  // all or nothing, so the arrays are sized for one m.  Nothing in the slots, x_prev, b_prev or rho is used before a
  // step writes it; comp is zero: every history empty
  Rollback<tsb_newton_s> undo(nw);
  tsb::LbfgsParams L{};
  int rc = alloc_once(nw, M1 * rows * 3, &L.s, st, refusal);
  if (rc == TSB_OK) rc = alloc_once(nw, M1 * rows * 3, &L.y, st, refusal);
  if (rc == TSB_OK) rc = alloc_once(nw, rows * 3, &L.x_prev, st, refusal);
  if (rc == TSB_OK) rc = alloc_once(nw, rows * 3, &L.b_prev, st, refusal);
  if (rc == TSB_OK) rc = alloc_once(nw, M1 * S, &L.rho, st, refusal);
  if (rc == TSB_OK) rc = alloc_once(nw, S, &L.comp, st, refusal, true);
  if (rc != TSB_OK) return rc;
  undo.commit();
  L.m = m;
  L.rows = int32_t(rows);
  nw->lb = L;
  return TSB_OK;
}

}  // namespace

extern "C" {

int tsb_newton_lbfgs_step(tsb_newton_t nw, float *x_dev, const float *anchor_dev, const float *weight_dev,
                          const tsb_terms_t *terms, const tsb_newton_lbfgs_options_t *opt,
                          tsb_newton_lbfgs_sphere_t *records_out_dev, void *stream) {
  if (!nw) return TSB_E_INVALID;
  int rc = newton_pointers_check(nw, x_dev, anchor_dev, weight_dev, terms, opt);
  if (rc != TSB_OK) return rc;
  const std::string rule = lbfgs_rule_error(*opt);
  if (!rule.empty()) return fail(nw, TSB_E_INVALID, rule);
  if (nw->lb.m && opt->m != nw->lb.m)
    return fail(nw, TSB_E_INVALID, "m = " + std::to_string(opt->m) + " but this workspace's L-BFGS history was sized for m = " +
                                       std::to_string(nw->lb.m) + " by its first L-BFGS step");
  tsb_pcg_t s = nw->s;
  if (const char *m = check_terms(s->h, s->psd, *terms)) return fail(nw, TSB_E_INVALID, m);
  if (s->sgs || s->coarse)     // H0 is the block-Jacobi preconditioner alone
    return fail(nw, TSB_E_INVALID, "the L-BFGS step takes H0 from block Jacobi: not on a workspace with the SGS preconditioner "
                                   "(tsb_pcg_enable_sgs) or the coarse space (tsb_pcg_enable_coarse)");
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail(nw, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = lbfgs_alloc(nw, opt->m, st);
  if (rc != TSB_OK) return rc;
  const tsb::NewtonParams &W = nw->W;
  const tsb::ProxParams pp{x_dev, anchor_dev, weight_dev, nullptr};
  const tsb::ProxParams *prox = anchor_dev ? &pp : nullptr;
  const tsb::LbfgsRule r{opt->gtol, opt->sigma, opt->eta, opt->curv_eps, opt->n_alpha};
  // b = -grad (prox: b -= w (x - y)), frozen spheres' b = 0; H0 = P from the diagonal blocks with the shift w_c (prox)
  rc = newton_rhs(nw, x_dev, terms, prox, st);
  if (rc != TSB_OK) return rc;
  rc = tsb_pcg_set_blocks_ex(s, W.diag, opt->rel_floor, weight_dev, nullptr, st);
  if (rc != TSB_OK) return fail(nw, rc, s->err);
  // the direction, the line search at 2^-k, k < n_alpha, per sphere, the decision and the step
  cudaError_t e = tsb::launch_lbfgs_dir(s->P, W, nw->lb, r, x_dev, prox, st);
  if (e != cudaSuccess) return fail(nw, TSB_E_CUDA, std::string("lbfgs launch: ") + cudaGetErrorString(e));
  rc = tsb_line_search(s->h, x_dev, W.d, terms, W.alphas, opt->n_alpha, nw->delta, nullptr, W.sphere_delta, W.sphere_step, st);
  if (rc != TSB_OK) return fail(nw, rc, s->h->err);
  e = tsb::launch_lbfgs_decide(s->P, W, nw->lb, r, prox, records_out_dev, st);
  if (e == cudaSuccess) e = tsb::launch_sphere_axpy(s->P, x_dev, W.alpha_sphere, W.d, x_dev, st);
  if (e != cudaSuccess) return fail(nw, TSB_E_CUDA, std::string("lbfgs launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

/* ---- Assembled Hessian (tsb_hessian.cu) ---- */

int tsb_hessian_create(tsb_pcg_t s, const float *rest_xyz, const int32_t *tets, int32_t nele, tsb_hessian_t *out) {
  if (!out) return fail<tsb_hessian_s>(nullptr, TSB_E_INVALID, "out is null");
  *out = nullptr;
  if (!s) return fail<tsb_hessian_s>(nullptr, TSB_E_INVALID, "solver workspace is null");
  if (!rest_xyz || !tets) return fail<tsb_hessian_s>(nullptr, TSB_E_INVALID, "rest_xyz and tets must be non-null");
  const tsb_handle_t h = s->h;
  if (nele != h->info.nele)
    return fail<tsb_hessian_s>(nullptr, TSB_E_INVALID, "nele = " + std::to_string(nele) + " but the handle has " + std::to_string(h->info.nele) + " tets");
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail<tsb_hessian_s>(nullptr, TSB_E_CUDA, "cannot select the handle's CUDA device");
  int rc = refuse_capture<tsb_hessian_s>(nullptr, cudaStreamLegacy,
                                         "tsb_hessian_create allocates device memory and cannot run while a stream is being captured");
  if (rc != TSB_OK) return rc;
  tsb::HessPattern H;
  std::string err;
  rc = tsb::build_hessian_pattern(rest_xyz, tets, h->info.n, nele, h->lap_scale, H, err);
  if (rc != TSB_OK) return fail<tsb_hessian_s>(nullptr, rc, err);
  if (H.comp_label != h->comp_label || H.nnz != h->info.nnz)
    return fail<tsb_hessian_s>(nullptr, TSB_E_MESH, "the mesh's components or operator differ from the handle's: not the mesh it was created from");
  tsb::TetTables T;
  rc = tsb::build_tet_tables(rest_xyz, tets, h->info.n, nele, nullptr, T, err);
  if (rc != TSB_OK) return fail<tsb_hessian_s>(nullptr, rc, err);
  tsb_hessian_t hs = new tsb_hessian_s();
  hs->s = s;
  hs->device = h->device;
  hs->psd = s->psd;
  hs->nnzb = H.nnzb;
  tsb::HessParams &P = hs->P;
  const size_t ne = size_t(nele);
  Rollback<tsb_hessian_s> undo(hs, tsb_hessian_destroy);
  rc = device_array(hs, hs->crow, 0, H.crow.data(), H.crow.size());
  if (rc == TSB_OK) rc = device_array(hs, hs->col, 0, H.col.data(), H.col.size());
  if (rc == TSB_OK) rc = device_array(hs, P.w, 0, H.w.data(), H.w.size());
  if (rc == TSB_OK) rc = device_array(hs, P.tblk, 0, H.tblk.data(), H.tblk.size());
  if (rc == TSB_OK) rc = device_array(hs, P.inc_ptr, 0, T.inc_ptr.data(), T.inc_ptr.size());
  if (rc == TSB_OK) rc = device_array(hs, P.inc, 0, T.inc.data(), T.inc.size());
  if (rc == TSB_OK) rc = device_array(hs, P.kind, ne);
  if (rc == TSB_OK) rc = device_array(hs, P.blk, ne * tsb::kHessTetFloats);
  if (hs->psd) {                     // the projection's tets and rest inverses, a private operator
    if (rc == TSB_OK) rc = device_array(hs, P.op, ne * tsb::kPsdOpFloats);
    P.tets = s->Q.tets;
    P.B = s->Q.B;
  } else {
    if (rc == TSB_OK) rc = device_array(hs, P.tets, 0, T.tets.data(), T.tets.size());
    if (rc == TSB_OK) rc = device_array(hs, P.B, 0, T.B.data(), T.B.size());
  }
  if (rc != TSB_OK) return rc;
  undo.commit();
  P.crow = hs->crow;
  P.n = h->info.n; P.nele = nele;
  *out = hs;
  return TSB_OK;
}

void tsb_hessian_destroy(tsb_hessian_t hs) {
  if (!hs) return;
  DeviceGuard guard(hs->device);
  for (void *p : hs->allocs) cudaFree(p);
  delete hs;
}

const char *tsb_hessian_last_error(tsb_hessian_t hs) { return hs ? hs->err.c_str() : create_err<tsb_hessian_s>().c_str(); }

int64_t tsb_hessian_device_bytes(tsb_hessian_t hs) { return hs ? hs->device_bytes : 0; }

int tsb_hessian_pattern(tsb_hessian_t hs, int64_t *nnzb, int32_t *crow_dev_out, int32_t *col_dev_out, void *stream) {
  if (!hs) return TSB_E_INVALID;
  if (nnzb) *nnzb = hs->nnzb;
  DeviceGuard guard(hs->device);
  if (!guard.ok) return fail(hs, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaSuccess;
  if (crow_dev_out) e = cudaMemcpyAsync(crow_dev_out, hs->crow, (size_t(hs->P.n) + 1) * sizeof(int32_t), cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess && col_dev_out)
    e = cudaMemcpyAsync(col_dev_out, hs->col, size_t(hs->nnzb) * sizeof(int32_t), cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) return fail(hs, TSB_E_CUDA, std::string("pattern copy: ") + cudaGetErrorString(e));
  return TSB_OK;
}

int tsb_hessian_assemble(tsb_hessian_t hs, const float *x_dev, const tsb_terms_t *terms, float *values_dev, void *stream) {
  if (!hs) return TSB_E_INVALID;
  if (!x_dev || !terms || !values_dev) return fail(hs, TSB_E_INVALID, "x_dev, terms and values_dev must be non-null");
  if (const char *m = check_terms(hs->s->h, hs->psd, *terms)) return fail(hs, TSB_E_INVALID, m);
  DeviceGuard guard(hs->device);
  if (!guard.ok) return fail(hs, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaSuccess;
  if (hs->psd) {                     // the workspace's projection kernel, into this workspace's operator and activity
    tsb::PsdParams Q = hs->s->Q;
    Q.op = const_cast<float *>(hs->P.op);
    Q.kind = hs->P.kind;
    e = tsb::launch_psd_project(Q, x_dev, terms->order, terms->c3 != 0.f ? 1 : 0, st);
  }
  if (e == cudaSuccess) e = tsb::launch_hessian_blocks(hs->P, x_dev, terms->order, terms->c2, terms->c3, hs->psd, st);
  if (e == cudaSuccess) e = tsb::launch_hessian_gather(hs->P, terms->c1, values_dev, st);
  if (e != cudaSuccess) return fail(hs, TSB_E_CUDA, std::string("hessian launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

/* ---- Symmetric Gauss-Seidel preconditioner (tsb_sgs.cu) ---- */

int tsb_pcg_enable_sgs(tsb_pcg_t s, tsb_hessian_t hs) {
  if (!s) return TSB_E_INVALID;
  if (s->sgs) return fail(s, TSB_E_INVALID, "the symmetric Gauss-Seidel preconditioner is already enabled on this workspace");
  if (!hs) return fail(s, TSB_E_INVALID, "hs is null");
  if (hs->s != s) return fail(s, TSB_E_INVALID, "hs was created over another solver workspace");
  const tsb_handle_t h = s->h;
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  int rc = refuse_capture(s, cudaStreamLegacy, "tsb_pcg_enable_sgs allocates device memory and cannot run while a stream is being captured");
  if (rc != TSB_OK) return rc;
  const size_t n = size_t(h->info.n), S = size_t(s->P.n_components);
  std::vector<int32_t> crow(n + 1), col(size_t(hs->nnzb));
  cudaError_t e = cudaMemcpy(crow.data(), hs->crow, crow.size() * sizeof(int32_t), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && !col.empty()) e = cudaMemcpy(col.data(), hs->col, col.size() * sizeof(int32_t), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("pattern download: ") + cudaGetErrorString(e));
  tsb::PcgLists L;
  tsb::build_pcg_lists(h->comp_label, int32_t(S), L);
  int32_t big = 0;
  for (size_t c = 0; c < S; ++c)
    if (L.comp_off[c + 1] - L.comp_off[c] > L.comp_off[size_t(big) + 1] - L.comp_off[size_t(big)]) big = int32_t(c);
  const int32_t max_verts = S ? L.comp_off[size_t(big) + 1] - L.comp_off[size_t(big)] : 0;
  int limit = 0;
  e = tsb::sgs_configure(max_verts, &limit);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("sweep configuration: ") + cudaGetErrorString(e));
  if (max_verts > limit)
    return fail(s, TSB_E_INVALID, "component " + std::to_string(big) + " has " + std::to_string(max_verts) +
                                      " vertices; the sweep keeps a component's vector in one CTA's shared memory, at most " +
                                      std::to_string(limit) + " vertices on this device");
  tsb::SgsTables T;
  std::string err;
  rc = tsb::build_sgs_tables(crow, col, L, 0, T, err);
  if (rc != TSB_OK) return fail(s, rc, err);
  tsb::SgsParams G{};
  Rollback<tsb_pcg_s> undo(s);
  float *values = nullptr;
  int32_t *color = nullptr;
  rc = device_array(s, values, 9 * std::max<size_t>(col.size(), 1));
  if (rc == TSB_OK) rc = device_array(s, G.comp_off, 0, L.comp_off.data(), L.comp_off.size());
  if (rc == TSB_OK) rc = device_array(s, G.color_ptr, 0, T.color_ptr.data(), T.color_ptr.size());
  if (rc == TSB_OK) rc = device_array(s, G.color_off, 1, T.color_off.empty() ? nullptr : T.color_off.data(), T.color_off.size());
  if (rc == TSB_OK) rc = device_array(s, G.sched, 1, T.sched.empty() ? nullptr : T.sched.data(), T.sched.size());
  if (rc == TSB_OK) rc = device_array(s, G.lo_ptr, 0, T.lo_ptr.data(), T.lo_ptr.size());
  if (rc == TSB_OK) rc = device_array(s, G.hi_ptr, 0, T.hi_ptr.data(), T.hi_ptr.size());
  if (rc == TSB_OK) rc = device_array(s, G.lo, 2, T.lo.empty() ? nullptr : T.lo.data(), T.lo.size());
  if (rc == TSB_OK) rc = device_array(s, G.hi, 2, T.hi.empty() ? nullptr : T.hi.data(), T.hi.size());
  if (rc == TSB_OK) rc = device_array(s, color, 0, T.color.data(), T.color.size());
  if (rc != TSB_OK) return rc;       // the rollback leaves the workspace as it was
  undo.commit();
  G.values = values; G.crow = hs->crow; G.col = hs->col; G.max_verts = max_verts;
  s->G = G;
  s->sgs_values = values;
  s->sgs_color = color;
  s->sgs_n_colors = T.n_colors;
  s->sgs = hs;
  return TSB_OK;
}

int tsb_pcg_set_matrix(tsb_pcg_t s, const float *x_dev, const tsb_terms_t *terms, float *diag_out_dev, void *stream) {
  if (!s) return TSB_E_INVALID;
  if (!s->sgs) return fail(s, TSB_E_INVALID, "tsb_pcg_set_matrix needs a workspace after tsb_pcg_enable_sgs");
  if (!x_dev || !terms || !diag_out_dev) return fail(s, TSB_E_INVALID, "x_dev, terms and diag_out_dev must be non-null");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int rc = tsb_hessian_assemble(s->sgs, x_dev, terms, s->sgs_values, st);
  if (rc != TSB_OK) return fail(s, rc, s->sgs->err);
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaError_t e = tsb::launch_sgs_diag(s->G, s->P.n, diag_out_dev, st);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("diagonal launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

int tsb_pcg_apply_precond(tsb_pcg_t s, const float *r_dev, float *z_dev, void *stream) {
  if (!s) return TSB_E_INVALID;
  if (!s->sgs && !s->coarse)
    return fail(s, TSB_E_INVALID, "tsb_pcg_apply_precond needs a workspace after tsb_pcg_enable_sgs or tsb_pcg_enable_coarse");
  if (!r_dev || !z_dev) return fail(s, TSB_E_INVALID, "r_dev and z_dev must be non-null");
  if (r_dev == z_dev) return fail(s, TSB_E_INVALID, "z_dev must not be r_dev: r is read after z is written");
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaSuccess;
  if (s->sgs) e = tsb::launch_sgs_sweep(s->P, s->G, tsb::SgsSweep{r_dev, z_dev, nullptr, 0, 0, -1, nullptr, nullptr}, st);
  if (e == cudaSuccess && s->coarse) e = tsb::launch_coarse_restrict(s->P, s->co, r_dev, st);
  if (e == cudaSuccess && s->coarse) e = tsb::launch_coarse_apply(s->P, s->co, r_dev, z_dev, !s->sgs, st);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("preconditioner launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

/* ---- Affine coarse space (tsb_coarse.cu) ---- */

int tsb_pcg_enable_coarse(tsb_pcg_t s, const float *rest_xyz, const int32_t *tets, int32_t nele, float coarse_floor) {
  if (!s) return TSB_E_INVALID;
  if (s->coarse) return fail(s, TSB_E_INVALID, "the coarse space is already enabled on this workspace");
  if (!rest_xyz || !tets) return fail(s, TSB_E_INVALID, "rest_xyz and tets must be non-null");
  if (!(coarse_floor >= 0.f)) return fail(s, TSB_E_INVALID, "coarse_floor must be >= 0");
  const tsb_handle_t h = s->h;
  if (nele != h->info.nele)
    return fail(s, TSB_E_INVALID, "nele = " + std::to_string(nele) + " but the handle has " + std::to_string(h->info.nele) + " tets");
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  int rc = refuse_capture(s, cudaStreamLegacy, "tsb_pcg_enable_coarse allocates device memory and cannot run while a stream is being captured");
  if (rc != TSB_OK) return rc;
  tsb::TetTables T;
  std::string err;
  rc = tsb::build_tet_tables(rest_xyz, tets, h->info.n, nele, &h->comp_label, T, err);
  if (rc != TSB_OK) return fail(s, TSB_E_INVALID, err + " (tets must be the mesh the handle was created from)");
  tsb::PcgLists L;
  tsb::build_pcg_lists(h->comp_label, s->P.n_components, L);
  tsb::CoarseTables CT;
  tsb::build_coarse_tables(rest_xyz, T, h->comp_label, L, CT);
  tsb::CoarseParams co{};
  co.n_tchunks = int32_t(CT.tchunk.size() / 3); co.nele = nele; co.floor = coarse_floor;
  const size_t S = size_t(s->P.n_components);
  Rollback<tsb_pcg_s> undo(s);
  rc = device_array(s, co.Y, 1, CT.Y.empty() ? nullptr : CT.Y.data(), CT.Y.size());
  if (rc == TSB_OK) rc = device_array(s, co.rpart, 9 * std::max<size_t>(size_t(s->P.n_chunks), 1));
  if (rc == TSB_OK) rc = device_array(s, co.tchunk, 3, CT.tchunk.empty() ? nullptr : CT.tchunk.data(), CT.tchunk.size());
  if (rc == TSB_OK) rc = device_array(s, co.comp_tchunk, 0, CT.comp_tchunk.data(), CT.comp_tchunk.size());
  if (rc == TSB_OK) rc = device_array(s, co.tet, 1, CT.tet.empty() ? nullptr : CT.tet.data(), CT.tet.size());
  if (rc == TSB_OK) rc = device_array(s, co.tets, 4, CT.tets.empty() ? nullptr : CT.tets.data(), CT.tets.size());
  if (rc == TSB_OK) rc = device_array(s, co.B, 9, CT.B.empty() ? nullptr : CT.B.data(), CT.B.size());
  if (rc == TSB_OK) rc = device_array(s, co.epart, size_t(tsb::kCoarseUpper) * std::max<size_t>(size_t(co.n_tchunks), 1));
  if (rc == TSB_OK) rc = device_array(s, co.S, 6, CT.S.empty() ? nullptr : CT.S.data(), CT.S.size());
  if (rc == TSB_OK) rc = device_array(s, co.Einv, 81 * std::max<size_t>(S, 1));
  if (rc != TSB_OK) return rc;       // the rollback leaves the workspace as it was
  undo.commit();
  s->co = co;
  s->coarse = true;
  return TSB_OK;
}

int tsb_pcg_set_coarse(tsb_pcg_t s, const float *x_dev, const tsb_terms_t *terms, void *stream) {
  if (!s) return TSB_E_INVALID;
  if (!s->coarse) return fail(s, TSB_E_INVALID, "tsb_pcg_set_coarse needs a workspace after tsb_pcg_enable_coarse");
  if (!x_dev || !terms) return fail(s, TSB_E_INVALID, "x_dev and terms must be non-null");
  if (const char *m = check_terms(s->h, s->psd, *terms)) return fail(s, TSB_E_INVALID, m);
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  return coarse_form(s, x_dev, *terms, true, static_cast<cudaStream_t>(stream));
}

int tsb_pcg_coarse_matrix(tsb_pcg_t s, double *E_out_dev) {
  if (!s) return TSB_E_INVALID;
  if (!s->coarse) return fail(s, TSB_E_INVALID, "tsb_pcg_coarse_matrix needs a workspace after tsb_pcg_enable_coarse");
  if (!E_out_dev) return fail(s, TSB_E_INVALID, "E_out_dev must be non-null");
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  cudaError_t e = tsb::launch_coarse_factor(s->P, s->co, nullptr, E_out_dev, cudaStreamLegacy);
  if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("coarse launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

int tsb_pcg_sgs_colors(tsb_pcg_t s, int32_t *colors_out_dev, int32_t *n_colors_out) {
  if (!s) return TSB_E_INVALID;
  if (!s->sgs) return fail(s, TSB_E_INVALID, "tsb_pcg_sgs_colors needs a workspace after tsb_pcg_enable_sgs");
  if (n_colors_out) *n_colors_out = s->sgs_n_colors;
  if (!colors_out_dev) return TSB_OK;
  DeviceGuard guard(s->h->device);
  if (!guard.ok) return fail(s, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const cudaError_t e = cudaMemcpy(colors_out_dev, s->sgs_color, size_t(s->P.n) * sizeof(int32_t), cudaMemcpyDeviceToDevice);
  if (e != cudaSuccess) return fail(s, TSB_E_CUDA, std::string("colour copy: ") + cudaGetErrorString(e));
  return TSB_OK;
}

int tsb_energy_grad_host(tsb_handle_t h, const float *x_host, float c1, float c2, int32_t order, float gradH,
                         float *energy_out_host, float *grad_out_host, void *stream) {
  if (!h) return TSB_E_INVALID;
  if (!x_host || !energy_out_host) return fail(h, TSB_E_INVALID, "x_host and energy_out_host must be non-null");
  if (order != 2 && order != 4) return fail(h, TSB_E_INVALID, "order must be 2 or 4");
  DeviceGuard guard(h->device);
  if (!guard.ok) return fail(h, TSB_E_CUDA, "cannot select the handle's CUDA device");
  const size_t nb = size_t(h->info.n) * 3 * sizeof(float);
  if (!h->stage_x[0]) {
    int rc = TSB_OK;
    for (int k = 0; k < 2 && rc == TSB_OK; ++k) {
      rc = device_array(h, h->stage_x[k], size_t(h->info.n) * 3);
      if (rc == TSB_OK) rc = device_array(h, h->stage_grad[k], size_t(h->info.n) * 3);
      if (rc == TSB_OK) rc = device_array(h, h->stage_energy[k], 4);
    }
    if (rc != TSB_OK) return rc;
    cudaError_t e = cudaSuccess;
    for (int k = 0; k < 2 && e == cudaSuccess; ++k) {
      e = cudaStreamCreateWithFlags(&h->s_pipe[k], cudaStreamNonBlocking);
      if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_run[k], cudaEventDisableTiming);
      if (e == cudaSuccess) e = cudaEventCreateWithFlags(&h->ev_done[k], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("pipeline stream setup: ") + cudaGetErrorString(e));
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cap) != cudaSuccess) { cudaGetLastError(); cap = cudaStreamCaptureStatusNone; }
  const int k = int(h->host_calls & 1u);
  cudaError_t e;
  if (cap != cudaStreamCaptureStatusNone) {      // inside a stream capture: keep it linear on the caller's stream
    e = cudaMemcpyAsync(h->stage_x[k], x_host, nb, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("H2D copy: ") + cudaGetErrorString(e));
    const int rc = tsb_energy_grad(h, h->stage_x[k], c1, c2, order, gradH, nullptr, h->stage_energy[k],
                                   grad_out_host ? h->stage_grad[k] : nullptr, stream);
    if (rc != TSB_OK) return rc;
    e = cudaMemcpyAsync(energy_out_host, h->stage_energy[k], 3 * sizeof(float), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && grad_out_host) e = cudaMemcpyAsync(grad_out_host, h->stage_grad[k], nb, cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("D2H copy: ") + cudaGetErrorString(e));
    return TSB_OK;
  }
  ++h->host_calls;
  // stream k: upload (ordered after call i-2's download of the same buffers by stream order) ...
  cudaStream_t sk = h->s_pipe[k];
  e = cudaMemcpyAsync(h->stage_x[k], x_host, nb, cudaMemcpyHostToDevice, sk);
  // ... kernel, after the previous call's kernel on the other stream (the handle's counters are shared) ...
  if (e == cudaSuccess) e = cudaStreamWaitEvent(sk, h->ev_run[k ^ 1], 0);
  if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("H2D copy: ") + cudaGetErrorString(e));
  // pinned + mapped host memory has a device alias (UVA): the kernel stores the 3 floats there itself, one copy
  // less per call (looked up every call: the address may have been freed and reused as pageable memory)
  float *e_alias = nullptr;
  {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, energy_out_host) == cudaSuccess && a.type == cudaMemoryTypeHost && a.devicePointer)
      e_alias = static_cast<float *>(a.devicePointer);
    else
      cudaGetLastError();
  }
  float *e_dst = e_alias ? e_alias : h->stage_energy[k];
  const int rc = tsb_energy_grad(h, h->stage_x[k], c1, c2, order, gradH, nullptr, e_dst,
                                 grad_out_host ? h->stage_grad[k] : nullptr, sk);
  if (rc != TSB_OK) return rc;
  e = cudaEventRecord(h->ev_run[k], sk);
  // ... download; the caller's stream waits for it, so synchronising `stream` completes the call
  if (e == cudaSuccess && !e_alias)
    e = cudaMemcpyAsync(energy_out_host, h->stage_energy[k], 3 * sizeof(float), cudaMemcpyDeviceToHost, sk);
  if (e == cudaSuccess && grad_out_host) e = cudaMemcpyAsync(grad_out_host, h->stage_grad[k], nb, cudaMemcpyDeviceToHost, sk);
  if (e == cudaSuccess) e = cudaEventRecord(h->ev_done[k], sk);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(st, h->ev_done[k], 0);
  if (e != cudaSuccess) return fail(h, TSB_E_CUDA, std::string("D2H copy: ") + cudaGetErrorString(e));
  return TSB_OK;
}

int tsb_scale(const float *g_dev, int64_t count, float gradH, const float *gradH_dev, float *out_dev, void *stream) {
  if (!g_dev || !out_dev || count < 0) return fail<tsb_handle_s>(nullptr, TSB_E_INVALID, "tsb_scale: null pointer or negative count");
  if (count == 0) return TSB_OK;
  DeviceGuard guard(device_of(g_dev));
  cudaError_t e = tsb::launch_scale(g_dev, count, gradH, gradH_dev, out_dev, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail<tsb_handle_s>(nullptr, TSB_E_CUDA, std::string("scale launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

int tsb_grad_limit(float *grad_dev, int64_t count, float s_threshold, float s, float *work_dev, void *stream) {
  if (!grad_dev || !work_dev || count < 0) return fail<tsb_handle_s>(nullptr, TSB_E_INVALID, "tsb_grad_limit: null pointer or negative count");
  if (count == 0) return TSB_OK;
  DeviceGuard guard(device_of(grad_dev));
  cudaError_t e = tsb::launch_grad_limit(grad_dev, count, s_threshold, s, work_dev, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail<tsb_handle_s>(nullptr, TSB_E_CUDA, std::string("grad_limit launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

int tsb_adam_uniform_step(float *p_dev, const float *grad_dev, float *g1_dev, float *g2_dev, int64_t count, double lr,
                          double beta1, double beta2, int32_t step, double grad_limit, float *work_dev, void *stream) {
  if (!p_dev || !grad_dev || !g1_dev || !g2_dev || !work_dev || count < 0 || step < 1)
    return fail<tsb_handle_s>(nullptr, TSB_E_INVALID, "tsb_adam_uniform_step: null pointer, negative count or step < 1");
  if (count == 0) return TSB_OK;
  DeviceGuard guard(device_of(p_dev));
  cudaError_t e = tsb::launch_adam_uniform(p_dev, grad_dev, g1_dev, g2_dev, count, lr, beta1, beta2, step, grad_limit,
                                           work_dev, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail<tsb_handle_s>(nullptr, TSB_E_CUDA, std::string("adam_uniform launch: ") + cudaGetErrorString(e));
  return TSB_OK;
}

#ifdef TSB_TRACE
/* profiling build only: copy the [grid][kTraceSlots] phase stamps of the last launch to the host */
int tsb_trace_read(tsb_handle_t h, unsigned long long *out, int64_t count) {
  if (!h || !out) return TSB_E_INVALID;
  DeviceGuard guard(h->device);
  const int64_t have = int64_t(h->info.grid) * tsb::kTraceSlots;
  return cudaMemcpy(out, h->kp.trace, size_t(std::min(count, have)) * 8, cudaMemcpyDeviceToHost) == cudaSuccess ? TSB_OK : TSB_E_CUDA;
}
#endif

}  // extern "C"
