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

// Trust-region recurrences of one component (tsb_pcg_solve_tr), in preconditioner norm |v|_M^2 = v^T P^-1 v.  A separate
// array, allocated by a workspace's first trust-region solve, so PcgComp and the plain solves are unchanged.  The lead
// thread of the component's first chunk in the dir kernel writes pMp, dMp and dMd (the update kernel reads them in every
// chunk); the update kernel's lead writes step (the dir kernel's lead reads it).  32 bytes.
struct TrComp {
  double pMp;    // |p|_M^2 of the current direction
  double dMp;    // d^T M p
  double dMd;    // |d|_M^2 of the current iterate
  double step;   // the step the last update took along p: alpha, the boundary tau, or 0 when d did not move
};
static_assert(sizeof(TrComp) == 32, "TrComp must be 32 bytes");

struct TrParams {
  const float *radius;   // [n_components] Delta_c (+inf: no radius; NaN or <= 0: radius 0)
  TrComp *comp;          // [n_components]
};

// State of one component of the damped Newton step (tsb_newton_step).  The shift kernel writes mu, nu and init on a
// component's first step, the decision kernel mu, nu and status; the other kernels only read it.  32 bytes.
struct NewtonComp {
  double mu, nu;
  int32_t status;   // TSB_NEWTON_*
  int32_t init;     // mu initialised
  int32_t pad[2];
};
static_assert(sizeof(NewtonComp) == 32, "NewtonComp must be 32 bytes");

struct NewtonParams {
  float *b, *d;              // [n, 3]: -grad (zeroed on frozen components), the damped Newton direction
  float *diag;               // [2, n, 3]: tsb_hess_diag's planes
  float *shift;              // [n_components] fp32 mu_c handed to the solve
  float *alpha_sphere;       // [n_components] step taken
  const float *alphas;       // [TSB_LINE_MAX_ALPHA] 2^-k
  float *sphere_delta;       // [n_components][n_alpha][4] line search
  float *sphere_step;        // [n_components] inversion-free step over (0, 1]
  double *part;              // [n_chunks, 3] per-chunk partials: max (D_v)_ii, b.d, d.d
  NewtonComp *comp;          // [n_components]
};

// The proximal step's extra inputs (tsb_newton_prox_step), read by the PROX variants of the Newton kernels only.
struct ProxParams {
  const float *x, *anchor;   // [n, 3]: the point of the step and the anchor y
  const float *weight;       // [n_components] w_c
  double *part;              // [n_chunks] per-chunk partials of d.(x - y)
};

struct NewtonRule {           // the options the kernels read
  float tau, mu_min, mu_max, gtol, sigma, eta;
  int32_t n_alpha;
};

// Radius state of one component of the trust-region step (tsb_newton_tr_step), allocated by the first such step.  The
// radius kernel writes it on a component's first step after a reset, the decision kernel afterwards.  16 bytes.
struct TrState {
  double radius;    // Delta_c
  int32_t init;     // radius initialised
  int32_t pad;
};
static_assert(sizeof(TrState) == 16, "TrState must be 16 bytes");

struct NewtonTrParams {
  TrState *state;            // [n_components]
  float *radius;             // [n_components] fp32 Delta_c handed to the solve
  const TrComp *tr;          // [n_components] the solve's recurrences (|d|_M^2)
};

struct NewtonTrRule {         // the options the trust-region kernels read
  float gtol, radius_init, radius_min, radius_max, accept, eta;
};

struct NewtonBacktrack {      // the backtracking options of tsb_newton_tr_step_ex (tsb_newton_backtrack_t)
  float sigma;
  int32_t n_alpha;
};

struct SgsParams;   // tsb_sgs.cuh: with it, the launchers below apply the symmetric Gauss-Seidel sweep in place of P

// Affine coarse space of the two-level preconditioner P + Z E+ Z^T (tsb_pcg_enable_coarse; tsb_coarse.cu).  Per component
// c the 9 coarse unknowns are a 3 x 3 matrix A, (Z a)_i = A Y_i with Y_i = X_i - mean_c X (rest positions), so
// R = Z^T r = sum_i r_i Y_i^T, entry 3 a + b = sum_i r_i[a] Y_i[b].  E+ is the pseudo-inverse of E_c + shift_c (S_c (x) I3).
constexpr int kCoarseTetT = 256;   // tets per tet chunk (one CTA of the tet pass)
constexpr int kCoarseUpper = 45;   // unique entries of a symmetric 9 x 9: (a, b), a <= b, rows in order
struct CoarseParams {
  const float *Y;              // [rows][3] Y of every entry of PcgParams::vert
  double *rpart;               // [n_chunks][9] per-chunk partials of R (init / update / restrict write, dir / apply fold)
  const int32_t *tchunk;       // [3 * n_tchunks] (component, begin, end) into the component-sorted tet list
  const int32_t *comp_tchunk;  // [n_components + 1] first tet chunk of every component
  const int32_t *tet;          // [nele] tet ids grouped by component
  const int4 *tets;            // [nele] their vertex ids
  const float *B;              // [9][nele] their rest inverse Dm^-1
  double *epart;               // [n_tchunks][45] per-chunk partials of E_c (upper triangle)
  const double *S;             // [n_components][6] sum_i Y_i Y_i^T: 00 11 22 12 02 01
  double *Einv;                // [n_components][81] E+
  int32_t n_tchunks, nele;
  float floor;                 // eigenvalues <= floor * lambda_max give 0
};

cudaError_t launch_pcg_blocks(const PcgParams &s, const float *diag, float rel_floor, float *inv_out, cudaStream_t st);
// blocks D_v + shift[c] I (over the chunk table; orphan vertices unshifted)
cudaError_t launch_pcg_blocks_shift(const PcgParams &s, const float *diag, float rel_floor, const float *shift, float *inv_out,
                                    cudaStream_t st);
// r = b, z = P r, d = 0 and the first direction; leaves every component ACTIVE or ZERO_RHS
// (tr != nullptr: also initialises the trust-region recurrences; sgs != nullptr: z = M^-1 r by one sweep)
// (co != nullptr: the two-level preconditioner, z + Z E+ Z^T r, in the direction and in r.z)
cudaError_t launch_pcg_begin(const PcgParams &s, const float *b, float *d, const TrParams *tr, cudaStream_t st,
                             const SgsParams *sgs = nullptr, const CoarseParams *co = nullptr);
// after Hp = H p of iteration `iter` (0-based) is complete on the stream: curvature, update and next direction; with
// shift != nullptr the operator is H + shift[c] I; with tr != nullptr every component stays inside its radius; with
// sgs != nullptr z = M^-1 r by one sweep after the update
cudaError_t launch_pcg_step(const PcgParams &s, float *d, int iter, float rtol, const float *shift, const TrParams *tr,
                            cudaStream_t st, const SgsParams *sgs = nullptr, const CoarseParams *co = nullptr);
cudaError_t launch_pcg_count(const PcgParams &s, cudaStream_t st);
cudaError_t launch_pcg_records(const PcgParams &s, const float *b, const float *d, tsb_pcg_sphere_t *out, cudaStream_t st);
cudaError_t launch_sphere_axpy(const PcgParams &s, const float *x, const float *a, const float *d, float *out, cudaStream_t st);
// The Newton launchers below run the proximal variants when p != nullptr.
// b_c = 0 on frozen components (prox: b -= w (x - y)), per-chunk max (D_v)_ii
cudaError_t launch_newton_prep(const PcgParams &s, const NewtonParams &w, const ProxParams *p, cudaStream_t st);
// damped step: mu_c on a first step and the fp32 shift
cudaError_t launch_newton_shift(const PcgParams &s, const NewtonParams &w, const NewtonRule &r, const ProxParams *p,
                                cudaStream_t st);
// per-chunk b.d and d.d (and d.(x - y))
cudaError_t launch_newton_dots(const PcgParams &s, const NewtonParams &w, const ProxParams *p, cudaStream_t st);
// damped step: step choice, damping update, records (out may be null)
cudaError_t launch_newton_decide(const PcgParams &s, const NewtonParams &w, const NewtonRule &r, const ProxParams *p,
                                 tsb_newton_sphere_t *out, cudaStream_t st);
// trust-region step, after the preconditioner is set: b^T P b per component (sgs != nullptr: b^T M^-1 b), Delta_c on a
// first step, the fp32 radius
cudaError_t launch_newton_tr_radius(const PcgParams &s, const NewtonParams &w, const NewtonTrParams &t, const NewtonTrRule &r,
                                    cudaStream_t st, const SgsParams *sgs = nullptr);
// Coarse space (tsb_coarse.cu).  Per-chunk partials of E_c at x: exact (activity from det F in fp64; c2, c3 weights) or,
// with q != nullptr, the projected operators of q's last projection
struct PsdParams;
cudaError_t launch_coarse_tets(const CoarseParams &co, const float *x, int order, float c2, float c3, const PsdParams *q,
                               cudaStream_t st);
// E+ of every component from the partials, with E_c + shift_c (S_c (x) I3) (shift may be null: unshifted); with
// E_out != nullptr the unshifted E_c (81 per component) goes there instead and E+ is left as it is
cudaError_t launch_coarse_factor(const PcgParams &s, const CoarseParams &co, const float *shift, double *E_out, cudaStream_t st);
// the R partials of v, per chunk
cudaError_t launch_coarse_restrict(const PcgParams &s, const CoarseParams &co, const float *v, cudaStream_t st);
// z = P r + Z E+ Z^T r (jacobi) or z += Z E+ Z^T r (after the sweep wrote z), on the vertices of the chunk table; the R
// partials of r must be in place (launch_coarse_restrict)
cudaError_t launch_coarse_apply(const PcgParams &s, const CoarseParams &co, const float *r, float *z, bool jacobi, cudaStream_t st);
// trust-region step: acceptance, radius update, records (out may be null); bt != nullptr: a rejected step is backtracked
// along the line search's n_alpha step sizes (tsb_newton_tr_step_ex)
cudaError_t launch_newton_tr_decide(const PcgParams &s, const NewtonParams &w, const NewtonTrParams &t, const NewtonTrRule &r,
                                    const ProxParams *p, const NewtonBacktrack *bt, tsb_newton_tr_sphere_t *out, cudaStream_t st);

}  // namespace tsb
