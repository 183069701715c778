// Device-side state and launchers of the per-sphere L-BFGS step (tsb_lbfgs.cu; tsb_newton_lbfgs_step), used by
// tsb_capi.cu.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/tssplat_b200.h"
#include "tsb_solver.cuh"

namespace tsb {

constexpr int kLbfgsThreads = 512;   // threads of the direction kernel's CTA, which owns one sphere

// L-BFGS state of one component.  The direction kernel writes the ring (head, count), the pair and clearing flags and
// the dots; the decision kernel reads them and writes moved, and clears count when no step is found.  64 bytes.
struct LbfgsComp {
  double bb;         // |b_c|^2                                  (direction writes, decision reads)
  double bd;         // b.d                                      (direction writes, decision reads)
  double dd;         // |d|^2                                    (direction writes, decision reads)
  double dx;         // d.(x - y), proximal step only            (direction writes, decision reads)
  int32_t head;      // ring slot the next pair goes to, in [0, m + 1)
  int32_t count;     // pairs held, <= m
  int32_t moved;     // 1: the last step moved the sphere, so x_prev and b_prev give a pair
  int32_t pair;      // -1 no pair this step, 0 rejected by the curvature test, 1 kept
  int32_t cleared;   // 1: the history was cleared this step
  int32_t pad[3];
};
static_assert(sizeof(LbfgsComp) == 64, "LbfgsComp must be 64 bytes");

struct LbfgsParams {
  float *s, *y;        // [m + 1][rows][3] pair slots, indexed by the entry of PcgParams::vert
  float *x_prev;       // [rows][3] x at the last direction
  float *b_prev;       // [rows][3] b at the last direction
  double *rho;         // [n_components][m + 1] 1 / s_i.y_i per slot
  LbfgsComp *comp;     // [n_components]
  int32_t m, rows;
};

struct LbfgsRule {      // the options the kernels read
  float gtol, sigma, eta, curv_eps;
  int32_t n_alpha;
};

// The direction of every component after b (tsb_newton_prep) and P (tsb_pcg_set_blocks_ex) are in place: pair update,
// two-loop recursion, fallback to P b, x_prev / b_prev and the dots.  p != nullptr: the proximal variant.
cudaError_t launch_lbfgs_dir(const PcgParams &s, const NewtonParams &w, const LbfgsParams &l, const LbfgsRule &r,
                             const float *x, const ProxParams *p, cudaStream_t st);
// Step choice, history clearing and records (out may be null), after the line search.
cudaError_t launch_lbfgs_decide(const PcgParams &s, const NewtonParams &w, const LbfgsParams &l, const LbfgsRule &r,
                                const ProxParams *p, tsb_newton_lbfgs_sphere_t *out, cudaStream_t st);

}  // namespace tsb
