/* tssplat_b200 -- C ABI of the H100-native (sm_90a) geometry-energy hot path of TetSphere Splatting.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types.  Every entry point
 * names the reference interface it replaces (paths relative to the reference checkout,
 * gmh14/tssplat @ 0241e9e3).  The reference-side binding a maintainer would add is shown in
 * INTEGRATION.md; the in-repo Python binding is tssplat_b200/_capi.py (ctypes).
 *
 * All device pointers are CUDA device pointers on the handle's device.  `stream` is a
 * cudaStream_t passed as void* (NULL = legacy default stream).  Every function returns 0 on
 * success and a negative TSB_E_* code on failure; tsb_last_error() gives the message.
 * A handle is not re-entrant (it owns scratch buffers), exactly like the reference's TetSpheres
 * object (tssplat_ext/tet_spheres/tet_spheres.h:37).
 */
#ifndef TSSPLAT_B200_H_
#define TSSPLAT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TSB_VERSION 13
#define TSB_LINE_MAX_ALPHA 8   /* step sizes one tsb_line_search call may evaluate */

enum {
  TSB_OK = 0,
  TSB_E_INVALID = -1,   /* bad argument (null pointer, order not in {2,4}, sizes <= 0, ...)      */
  TSB_E_MESH = -2,      /* bad mesh: index out of range, zero-volume rest tet, non-manifold face */
  TSB_E_CUDA = -3,      /* a CUDA runtime call failed                                            */
  TSB_E_NOMEM = -4
};

typedef struct tsb_handle_s *tsb_handle_t;

typedef struct {
  int32_t warps_per_cta;    /* 0 = library default (16, one persistent CTA per SM); 8 = two CTAs per SM */
  int32_t laplacian_scale;  /* 0 = unscaled tet-graph Laplacian (what the reference requests:
                               tet_spheres.cpp:148 passes (1, 0)); 1 = rows divided by #nbrs    */
  int32_t ring_slots;       /* per-warp TMA ring depth in chunks of 6 cells: 0 = default (2); 2..8   */
  int32_t force_global;     /* 1: gather u/x from global memory instead of staging components in
                               shared memory (the mode used for components too large to stage)   */
  int32_t tet_cost_x100;    /* load-balance weight of one tet vs one operator entry, x100 (0 = default) */
  int32_t enable_amips;     /* 1: also keep the per-tet rest inverses (48 B/tet) so that tsb_energy_grad_ex
                               may add the AMIPS term; 0 (default): c3 must be 0                    */
  int32_t deterministic;    /* 1: bitwise repeatable gradient, also with inverted tets and AMIPS (see
                               tsb_energy_grad); costs a second launch and 64 B/tet of device memory */
  int32_t reserved[1];
} tsb_options_t;

/* Energy terms of tsb_energy_grad_ex.  c3 weighs the AMIPS term that BASELINE.json's north_star names:
 *   sum over tets with det F > 0 of  tr(F^T F) / (3 det(F)^(2/3)) - 1     (conformal AMIPS, Fu et al. 2015)
 * THE REFERENCE HAS NO SUCH TERM (nothing in the reference tree computes it: SURVEY.md F1), so there is no
 * reference oracle for it: it is verified against two fp64 restatements, finite differences and its known
 * answers (0 at rest and under similarity maps), never "against the reference".  Default off. */
typedef struct {
  float c1, c2;
  int32_t order;            /* 2 or 4 */
  float c3;                 /* AMIPS coefficient; 0 = exactly tsb_energy_grad */
  int32_t reserved[4];
} tsb_terms_t;

typedef struct {
  int32_t n;                /* vertices                                                          */
  int32_t nele;             /* tets                                                              */
  int32_t n_components;     /* connected components (= tet-spheres)                              */
  int32_t grid;             /* persistent CTAs per launch                                        */
  int32_t warps_per_cta;
  int32_t ctas_per_sm;
  int32_t mode_global;      /* 0 = components staged in shared memory, 1 = global gathers        */
  int32_t smem_bytes;       /* dynamic shared memory per CTA                                     */
  int32_t ring_slots;
  int32_t n_segments;       /* (CTA, component) work pieces                                      */
  int32_t n_boundary_faces;
  int32_t max_component_vertices;
  int64_t nnz;              /* off-diagonal entries of M = G^T L^T L G (per coordinate)          */
  int64_t nnz_padded;       /* entries stored in the row blocks (incl. padding)                  */
  int64_t device_bytes;     /* bytes of device memory owned by the handle                        */
  int64_t stream_bytes;     /* bytes one launch reads+writes: plan streams + rest + x + grad     */
} tsb_info_t;

/* Replaces TetSpheres::TetSpheres(int nv, double*, int ntet, int*) + TetSpheres::init
 * (tssplat_ext/tet_spheres/tet_spheres.cpp:119-126,140-203) and the libpgo operator builders it
 * calls (:148-149): builds the rows of M = G^T L^T L G (fp64, rounded to fp32 like :43-45), the
 * per-tet 1/det(Dm), and the per-warp work streams on the host, and uploads them to `device`.  rest_xyz: host float32 [3n] REST positions; tets: host int32
 * [4*nele], 0-based.  opt may be NULL. */
int tsb_create(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele,
               const tsb_options_t *opt, int device, tsb_handle_t *out);

/* Replaces TetSpheres::~TetSpheres (tet_spheres.cpp:128-138); frees everything (no leaks). */
void tsb_destroy(tsb_handle_t h);

/* Message of the last failure on this handle (h may be NULL: last tsb_create failure). */
const char *tsb_last_error(tsb_handle_t h);

int tsb_get_info(tsb_handle_t h, tsb_info_t *info);

/* THE HOT PATH.  Replaces tet_spheres_smooth_barrier + tet_spheres_smooth_barrier_backward
 * (tssplat_ext/tet_spheres/tet_spheres_cuda.cu:118-195 and :197-263: 5 cuSPARSE SpMVs, 2 kernels,
 * 3 cuBLAS calls and 3 host syncs) with ONE kernel launch and no host sync:
 *   energy_out[0] = c1 * 1/2 x^T G^T L^T L G x + c2 * sum_t max(-det F_t,0)^order
 *   energy_out[1] = 1/2 x^T G^T L^T L G x    energy_out[2] = sum_t max(-det F_t,0)^order
 *   grad_out      = gradH * d energy_out[0] / d x          ([n,3] fp32, fully overwritten)
 * x_dev: device float32 [3n], contiguous.  gradH_dev: optional device float (0-dim tensor's
 * data pointer); when non-NULL it multiplies gradH (so pass gradH = 1).  grad_out_dev may be NULL
 * (energy only: replaces the forward alone).  order must be 2 or 4 (the reference silently
 * returns zeros otherwise: cu:57-63).  One launch may be in flight per handle at a time (the handle
 * owns counters and scratch, like the reference's TetSpheres: tet_spheres.h:37); launches on one
 * stream are chained with programmatic dependent launch.  Results are bitwise repeatable when no tet
 * is inverted; inverted tets add their barrier gradient with red.global.add.f32 (order-dependent
 * rounding in the affected vertices only).
 * Deterministic handles (tsb_options_t.deterministic = 1): every contributing tet (inverted, or any tet
 * with J > 0 when the AMIPS term is on) stores its corner vectors in handle scratch, and a second
 * kernel on the same stream adds them to each vertex in a fixed order; grad_out_dev == NULL runs the
 * energy kernel alone.  The energies and the gradient are then a pure function of (plan, x, the
 * coefficients, gradH): bitwise identical across launches, streams, CUDA-graph replays and handles
 * created from the same mesh with the same options, for tsb_energy_grad, tsb_energy_grad_ex and
 * tsb_energy_grad_host alike.  The energies, and the gradient rows no contributing tet touches, are
 * bitwise those of a default handle with the same options.  The guarantee holds for one handle
 * configuration only: warps_per_cta, force_global (or a mesh that needs global gathers) and
 * ring_slots change the plan, and with it the summation order and the tets' vertex order. */
int tsb_energy_grad(tsb_handle_t h, const float *x_dev, float c1, float c2, int32_t order,
                    float gradH, const float *gradH_dev, float *energy_out_dev,
                    float *grad_out_dev, void *stream);

/* tsb_energy_grad plus the optional AMIPS term.  energy_out_dev: device float32 [4] = total, smoothness,
 * barrier, AMIPS (unweighted sums; total = c1*smooth + c2*barrier + c3*amips).  With terms->c3 == 0 the launch
 * is the very kernel tsb_energy_grad runs.  c3 != 0 needs a handle created with enable_amips = 1; its gradient
 * is added with red.global.add.f32 for every tet (order-dependent rounding), except on a deterministic handle. */
int tsb_energy_grad_ex(tsb_handle_t h, const float *x_dev, const tsb_terms_t *terms, float gradH,
                       const float *gradH_dev, float *energy_out_dev, float *grad_out_dev, void *stream);

/* Geometry statistics of one connected component (= one tet-sphere), from tsb_energy_grad_spheres.  40 bytes. */
typedef struct {
  double smooth;        /* 1/2 u^T M u restricted to the component's rows (unweighted, like energy_out[1])     */
  double barrier;       /* sum over its tets of max(-J,0)^order                                                 */
  double amips;         /* sum of the AMIPS term over its J > 0 tets; 0 unless terms->c3 != 0                   */
  float min_J;          /* smallest det F over its tets (the kernel's fp32 J, the value the barrier tests)      */
  int32_t n_inverted;   /* tets with J < 0 (exactly the tets that contribute to the barrier)                    */
  int32_t n_tets;       /* tets of the component                                                                 */
  int32_t first_vertex; /* its lowest vertex id: identifies the component in the caller's numbering              */
} tsb_sphere_stats_t;

/* tsb_energy_grad_ex plus per-sphere statistics: the same launch (same argument checks, same energy_out_dev and
 * grad_out_dev, which may be NULL) also writes one tsb_sphere_stats_t per connected component to spheres_out_dev
 * (device memory, [info.n_components], required: NULL is TSB_E_INVALID).  Records are in component order, which is
 * the order of the components' lowest vertex ids (so for spheres concatenated one after the other, record k is
 * sphere k); vertices no tet references belong to no record.  Every record is rewritten by every call; no host
 * sync.  The per-component sums are folded in fp64 in a fixed order, so the records are a pure function of (plan,
 * x, order, c3 != 0): bitwise identical across launches and CUDA-graph replays, on default and deterministic
 * handles, with or without grad_out_dev.  Summed over the components they give energy_out's terms up to fp64
 * rounding; energy_out itself may differ from tsb_energy_grad_ex's by one fp32 ulp (the fp64 partials are summed
 * per sphere first), and grad_out is computed exactly as there.
 * Cost: per-segment warp reductions in the energy kernel plus one small kernel (DESIGN.md section 5). */
int tsb_energy_grad_spheres(tsb_handle_t h, const float *x_dev, const tsb_terms_t *terms, float gradH,
                            const float *gradH_dev, float *energy_out_dev, float *grad_out_dev,
                            tsb_sphere_stats_t *spheres_out_dev, void *stream);

/* Hessian-vector product of the smoothness and barrier energy (no counterpart in the reference):
 *   hv_out   = gradH * (*gradH_dev) * H(x) v       ([n,3] fp32, fully overwritten, required)
 *   curv_out = v^T H v as { c1*vMv + c2*vHbv, vMv, vHbv }   (optional device float[3]; NOT scaled by gradH)
 * with H(x) = c1 M + c2 sum_t H_t(x): M = G^T L^T L G (the smoothness Hessian: 1/2 x^T M x has Hessian M), and H_t the
 * Hessian of max(-J_t, 0)^order, nonzero only for tets whose fp32 J (the value tsb_energy_grad tests) is negative.
 * vMv = v^T M v and vHbv = sum_t v^T H_t v.  H_t is the exact, indefinite tet Hessian (tsb_pcg_hvp_psd multiplies by its
 * PSD projection).
 * The AMIPS term is NOT part of the product: tsb_hvp differentiates c1*smooth + c2*barrier only, also on handles
 * created with enable_amips (tsb_hvp_ex below adds it).  x_dev, v_dev: device float32 [3n], contiguous; order 2 or 4;
 * vertices no tet references get zero rows.  The launch streams the same plan as tsb_energy_grad (one kernel, plus the
 * gather on deterministic handles) and works on every handle: it leaves the handle's scratch as the next
 * tsb_energy_grad expects, so the two may be chained on one stream.  Rows no inverted tet touches are bitwise
 * repeatable on every handle (and equal across default and deterministic handles of the same options); inverted tets
 * add their H_t v with red.global.add.f32 on a default handle, and through the deterministic gather on a deterministic
 * handle, where hv and curv are then bitwise identical across launches, streams and CUDA-graph replays.  DESIGN.md
 * section 5. */
int tsb_hvp(tsb_handle_t h, const float *x_dev, const float *v_dev, float c1, float c2, int32_t order,
            float gradH, const float *gradH_dev, float *hv_out_dev, float *curv_out_dev, void *stream);

/* tsb_hvp plus the AMIPS term: the Hessian-vector product of what tsb_energy_grad_ex differentiates.
 *   hv_out   = gradH * (*gradH_dev) * (c1 M + c2 sum_t H_t + c3 sum_t H_a,t) v      ([n,3] fp32, required)
 *   curv_out = { c1*vMv + c2*vHbv + c3*vHav, vMv, vHbv, vHav }   (optional device float[4]; NOT scaled by gradH)
 * with c1, c2, c3, order from *terms (required), and H_a,t the exact (indefinite) Hessian of the tet's AMIPS term
 * psi = tr(F^T F) / (3 J^(2/3)) - 1, nonzero only for tets whose fp32 J is positive (the tets whose AMIPS gradient
 * tsb_energy_grad_ex adds); vHav = sum_t v^T H_a,t v.  terms->c3 != 0 needs a handle created with enable_amips = 1
 * (TSB_E_INVALID otherwise, as tsb_energy_grad_ex).  With terms->c3 == 0 the launch is the very kernel tsb_hvp runs:
 * hv and curv[0..2] are bitwise tsb_hvp's, and curv[3] = 0.  With c3 != 0 every tet with J > 0 adds its H_a v with
 * red.global.add.f32 on a default handle (order-dependent rounding) and through the deterministic gather on a
 * deterministic handle, where hv and curv are bitwise identical across launches, streams and CUDA-graph replays.  Like
 * tsb_hvp it leaves the handle's scratch re-armed, so it chains with tsb_energy_grad(_ex) on one stream. */
int tsb_hvp_ex(tsb_handle_t h, const float *x_dev, const float *v_dev, const tsb_terms_t *terms, float gradH,
               const float *gradH_dev, float *hv_out_dev, float *curv_out_dev, void *stream);

/* Line search along a direction (no counterpart in the reference): the energy change at up to TSB_LINE_MAX_ALPHA step
 * sizes and the largest step before a tet inverts, in one pass over the plan.
 *   delta_out[k]  = { c1*ds + c2*db + c3*da, ds, db, da }      (device float [n_alpha][4], required)
 * where ds, db, da are the changes E_t(x + alpha_k d) - E_t(x) of the unweighted smoothness, barrier and AMIPS terms of
 * tsb_energy_grad_ex (da = 0 when terms->c3 == 0), computed as differences, never as two energies subtracted:
 * ds = alpha u^T M d + 1/2 alpha^2 d^T M d with u = x - X, and per tet from J(alpha) = det F(x + alpha d), a cubic, and
 * |F + alpha dF|^2, a quadratic.  A tet contributes AMIPS at alpha exactly when its fp32 J(alpha) > 0.
 *   step_out[0]   = the smallest alpha in (0, alpha_max], alpha_max = max_k alpha_k, at which a real tet whose fp32
 *                   J(x) > 0 reaches J = 0 (the first root of its cubic, also when the cubic comes back above 0 before
 *                   alpha_max); +inf if there is none or alpha_max <= 0.  Inverted tets are ignored.  The kernel's own
 *                   cubic is >= 0 at the returned value.  (optional device float [1])
 * Per sphere (optional, device memory, component order as tsb_energy_grad_spheres): sphere_delta_out
 * [n_components][n_alpha][4] and sphere_step_out [n_components], from fp64 per-sphere sums; delta_out is the
 * fixed-order fp64 sum of those sums rounded once, and step_out their minimum.  Vertices no tet references belong to no
 * sphere.  x_dev, d_dev: device float32 [3n]; alpha_dev: device float32 [n_alpha], 1 <= n_alpha <= TSB_LINE_MAX_ALPHA,
 * read on the device (a captured CUDA graph can be replayed with new step sizes).  c1, c2, order, c3 from *terms, with
 * tsb_energy_grad_ex's rules.  There are no atomics and no per-vertex output: every output is a pure function of (plan,
 * x, d, alpha, terms), bitwise identical across launches, streams, CUDA-graph replays, and default and deterministic
 * handles of the same options.  The line search uses no device memory of its own (its records reuse the per-sphere
 * statistics' scratch) and leaves the handle's scratch as tsb_energy_grad(_ex) and tsb_hvp(_ex) expect, so it chains
 * with them on one stream.  Three launches: the energy kernel's LINE variant and two small fold kernels.
 * Argument errors (TSB_E_INVALID, nothing launched): n_alpha outside [1, TSB_LINE_MAX_ALPHA], a null x_dev, d_dev,
 * alpha_dev, delta_out_dev or terms, an order other than 2 or 4, terms->c3 != 0 on a handle without enable_amips.
 * DESIGN.md section 5, "Line search". */
int tsb_line_search(tsb_handle_t h, const float *x_dev, const float *d_dev, const tsb_terms_t *terms,
                    const float *alpha_dev, int32_t n_alpha, float *delta_out_dev, float *step_out_dev,
                    float *sphere_delta_out_dev, float *sphere_step_out_dev, void *stream);

/* Per-vertex 3x3 diagonal blocks of the Hessian of what tsb_hvp_ex differentiates (no counterpart in the reference),
 * for block-Jacobi preconditioning:
 *   diag_out = gradH * (*gradH_dev) * D      (device float32 [2][n][3], fully overwritten, required)
 * where D_i is the 3x3 block of H(x) = c1 M + c2 sum_t H_t + c3 sum_t H_a,t at vertex i (the H of tsb_hvp_ex):
 * plane 0 holds (H_xx, H_yy, H_zz) of each vertex, plane 1 (H_yz, H_xz, H_xy).  The smoothness part is c1 M_ii I
 * (M = M1 (x) I3).  A tet with fp32 J < 0 adds, at each corner k, the rank-1 block p (p-1) (-J)^(p-2) g_k g_k^T
 * (g_k = dJ/dx_k); with c3 != 0 a tet with fp32 J > 0 adds the exact AMIPS block of its corner, which may be indefinite
 * far from rest.  Vertices no tet references get zero rows in both planes.  c1, c2, order, c3 from *terms with
 * tsb_hvp_ex's rules.  Default handle: one launch; the rows are stored, then active tets add their six entries per
 * corner with red.global.add.f32 (order-dependent rounding in their vertices).  Deterministic handle: one launch and
 * one deterministic gather per plane; the output is then bitwise identical across launches, streams, CUDA-graph replays
 * and handles with the same options, and rows no active tet touches are bitwise those of a default handle.  Uses no
 * device memory of its own and leaves the handle's scratch re-armed, so it chains with tsb_energy_grad(_ex),
 * tsb_hvp(_ex) and tsb_line_search on one stream.  Argument errors (TSB_E_INVALID, nothing launched): a null terms,
 * x_dev or diag_out_dev, an order other than 2 or 4, terms->c3 != 0 on a handle without enable_amips.
 * DESIGN.md section 5, "Hessian diagonal". */
int tsb_hess_diag(tsb_handle_t h, const float *x_dev, const tsb_terms_t *terms, float gradH, const float *gradH_dev,
                  float *diag_out_dev, void *stream);

/* ---- Newton-CG solve: per-sphere preconditioned CG on the device (no counterpart in the reference) --------------
 * Spheres share no vertices, so the Hessian H(x) of tsb_hvp_ex is block diagonal by connected component.  tsb_pcg_solve
 * runs block-Jacobi preconditioned, truncated (Steihaug) conjugate gradients on every block independently -- each
 * sphere its own alpha, beta, residual test and negative-curvature test -- with all spheres batched in the same
 * launches and every scalar in device memory: no device-to-host read inside an iteration.  DESIGN.md section 5,
 * "Newton-CG solve".
 *
 * A workspace is a separate object sized from a handle (which must outlive it); creating one changes nothing about the
 * handle (tsb_get_info and the plan stay as they are).  It owns the component vertex lists (the non-orphan vertex ids
 * grouped by component, ascending inside a component, components in the order of tsb_energy_grad_spheres), a chunk
 * table of <= 256 vertices per chunk, the vectors r, z, p, Hp, the inverse preconditioner blocks, per-chunk fp64
 * partial sums and the per-component state.  Device memory, reported by tsb_pcg_device_bytes:
 *   72 n + 4 rows + 36 chunks + 64 n_components + 4 (n_components + 1) + 4   bytes
 * (rows = vertices some tet references, chunks = sum over components of ceil(vertices / 256)).  Like a handle, a
 * workspace serves one stream at a time. */
typedef struct tsb_pcg_s *tsb_pcg_t;
int tsb_pcg_create(tsb_handle_t h, tsb_pcg_t *out);
void tsb_pcg_destroy(tsb_pcg_t s);
const char *tsb_pcg_last_error(tsb_pcg_t s);   /* s may be NULL: last tsb_pcg_create failure */
int64_t tsb_pcg_device_bytes(tsb_pcg_t s);

/* Sets the preconditioner from the diagonal blocks of tsb_hess_diag (diag_dev: device float32 [2][n][3]; NULL = the
 * identity, which is also what a new workspace holds).  One kernel, one thread per vertex: the symmetric 3x3 block is
 * diagonalised in fp64 registers (cyclic Jacobi), its eigenvalues are clamped from below to rel_floor * lambda_max and
 * the block is inverted; a block with lambda_max <= 0 (a vertex no tet references, or one with only negative curvature)
 * becomes the zero block, so that vertex does not move.  inv_out_dev (optional, device float32 [n][6]) receives the
 * inverse blocks as (xx, yy, zz, yz, xz, xy) per vertex.  No host sync. */
int tsb_pcg_set_blocks(tsb_pcg_t s, const float *diag_dev, float rel_floor, float *inv_out_dev, void *stream);

enum {
  TSB_PCG_MAXITER = 0,        /* max_iter products used, residual test not met                         */
  TSB_PCG_CONVERGED = 1,      /* |r_c| <= rtol |b_c|                                                    */
  TSB_PCG_NEGCURV = 2,        /* p^T H p <= 0 at a later direction: d_c is the iterate reached before it */
  TSB_PCG_NEGCURV_FIRST = 3,  /* p^T H p <= 0 at the first direction: d_c = P b_c                        */
  TSB_PCG_ZERO_RHS = 4,       /* |b_c| = 0: d_c = 0                                                      */
  TSB_PCG_BOUNDARY = 5,       /* tsb_pcg_solve_tr only: the next iterate would leave the radius; d_c on the boundary */
  TSB_PCG_NEGCURV_BOUNDARY = 6 /* tsb_pcg_solve_tr only: p^T H p <= 0, followed to the boundary (tau P b_c at the first
                                 direction)                                                                         */
};

typedef struct {
  int32_t max_iter;         /* >= 1: Hessian-vector products at most                                                 */
  float rtol;               /* >= 0: a sphere stops at |r_c| <= rtol |b_c|                                           */
  int32_t check_every;      /* 0: enqueue exactly max_iter iterations, never touch the host (capturable in a CUDA graph;
                               stopped spheres idle); k > 0: enqueue k iterations at a time, then read one int32, the
                               number of spheres still active, and stop when it is 0                                  */
  int32_t reserved[5];
} tsb_pcg_options_t;

typedef struct {            /* one per component, in the component order of tsb_energy_grad_spheres; 32 bytes        */
  float rel_residual;       /* |r_c| / |b_c| of the returned d_c from the recurrence's residual (1 at NEGCURV_FIRST,
                               0 at ZERO_RHS)                                                                         */
  float b_dot_d;            /* b_c . d_c: with b = -grad, minus the directional derivative of a per-sphere Armijo test */
  float d_H_d;              /* sum of alpha^2 p^T H p = d_c^T H d_c up to CG rounding; 0 if no step was accumulated   */
  int32_t n_hvp;            /* products in which this component was still active                                      */
  int32_t status;           /* TSB_PCG_*                                                                              */
  int32_t first_vertex;     /* its lowest vertex id                                                                   */
  int32_t n_vertices;
  int32_t reserved;
} tsb_pcg_sphere_t;

/* Solves H(x) d = b on every component, H exactly what tsb_hvp_ex multiplies by with *terms (c3 != 0 needs a handle
 * created with enable_amips = 1).  x_dev, b_dev: device float32 [3n]; d_out_dev: device float32 [3n], fully overwritten
 * (zero on vertices no tet references); spheres_out_dev: optional device array [info.n_components]; iters_run_out:
 * optional host int32, the iterations enqueued.  Per component c, independently: r = b_c, z = P r, p = z; each
 * iteration forms alpha = r.z / p^T H p, stops at p^T H p <= 0 (returning the iterate so far, or P b_c at the first
 * direction), else d += alpha p, r -= alpha H p, stops at |r| <= rtol |b_c|, else z = P r, p = z + beta p.  A stopped
 * component's p is 0, so later products leave it untouched and its d_c is final.
 * Per iteration the stream sees the launches of tsb_hvp_ex on p (the gather follows on deterministic handles) and
 * three small kernels over the chunk table.  Dot products are accumulated in fp64 in a fixed order and there are no
 * floating-point atomics, so on a deterministic handle d and the records are bitwise identical across calls, streams
 * and CUDA-graph replays, and a component's result does not depend on the other components' right-hand sides.  (On a
 * default handle the products add active tets' contributions with red.global.add.f32, as tsb_hvp_ex does.)
 * Chains with every other call of the handle on one stream.
 * Argument errors (TSB_E_INVALID, nothing launched): a null x_dev, b_dev, d_out_dev, terms or opt, max_iter < 1,
 * rtol < 0 or NaN, check_every < 0, check_every > 0 on a stream that is being captured, an order other than 2 or 4,
 * terms->c3 != 0 on a handle without enable_amips. */
int tsb_pcg_solve(tsb_pcg_t s, const float *x_dev, const float *b_dev, const tsb_terms_t *terms,
                  const tsb_pcg_options_t *opt, float *d_out_dev, tsb_pcg_sphere_t *spheres_out_dev,
                  int32_t *iters_run_out, void *stream);

/* Per-sphere step: out_v = x_v + a[component of v] * d_v, vertices no tet references copied.  a_sphere_dev: device
 * float32 [info.n_components]; out_dev may alias x_dev.  One launch, no host sync. */
int tsb_sphere_axpy(tsb_pcg_t s, const float *x_dev, const float *a_sphere_dev, const float *d_dev, float *out_dev,
                    void *stream);

/* ---- Damped (Levenberg-Marquardt) solve: H + mu_c I per sphere --------------------------------------------------
 * shift_dev: device float32 [info.n_components], mu_c >= 0 per component in component order, read on the device (a
 * captured graph can be replayed with new shifts).  With shift_dev == NULL both calls are exactly tsb_pcg_set_blocks and
 * tsb_pcg_solve.
 *
 * tsb_pcg_set_blocks_ex: every vertex of component c gets the block D_v + mu_c I before the eigen-clamp-invert of
 * tsb_pcg_set_blocks (vertices no tet references keep the zero block; diag_dev == NULL gives the identity, unshifted).
 * One launch over the component chunk table.
 *
 * tsb_pcg_solve_ex: solves (H(x) + mu_c I) d = b_c on every component with tsb_pcg_solve's algorithm, rules and records.
 * The shift enters as p.(Hp + mu p) in the curvature and r -= alpha (Hp + mu p) in the residual update, both in fp32
 * with the same rounding; the Hessian-vector product launches are tsb_pcg_solve's.  H + mu_c I is positive definite
 * once mu_c exceeds minus the smallest eigenvalue of the component's H, and the solve then converges where the unshifted
 * one stops at negative curvature.  In the records d_H_d is d^T (H + mu_c I) d. */
int tsb_pcg_set_blocks_ex(tsb_pcg_t s, const float *diag_dev, float rel_floor, const float *shift_dev, float *inv_out_dev,
                          void *stream);
int tsb_pcg_solve_ex(tsb_pcg_t s, const float *x_dev, const float *b_dev, const tsb_terms_t *terms,
                     const tsb_pcg_options_t *opt, const float *shift_dev, float *d_out_dev,
                     tsb_pcg_sphere_t *spheres_out_dev, int32_t *iters_run_out, void *stream);

/* ---- Trust-region solve (Steihaug-Toint CG) ------------------------------------------------------------------------
 * Solves (H(x) + shift_c I) d = b_c on every component with tsb_pcg_solve_ex's algorithm, options, preconditioner, rules
 * and records (shift_dev may be NULL), inside a per-component radius: |d_c|_M <= Delta_c in the preconditioner norm
 * |v|_M^2 = v^T P^-1 v, P the clamped inverse blocks of tsb_pcg_set_blocks(_ex) (the norm in which the CG iterates'
 * length grows monotonically, so the first crossing is the one to stop at).  radius_dev: device float32
 * [info.n_components], Delta_c in component order, read on the device (+inf: no radius; NaN or <= 0: radius 0, d_c = 0).
 * Per component, in fp64 and without an extra vector pass, the lead CTA keeps
 *   pMp_0 = r.z,  dMp_0 = dMd_0 = 0;  after a step s along p: dMd += 2 s dMp + s^2 pMp, and then
 *   dMp = beta (dMp + s pMp),  pMp = r.z + beta^2 pMp
 * and with tau >= 0 solving |d + tau p|_M = Delta, formed as (Delta^2 - dMd) / (dMp + sqrt(dMp^2 + pMp (Delta^2 - dMd))):
 *   p^T (H + shift) p <= 0:                    d += tau p, NEGCURV_BOUNDARY (tau P b_c at the first direction);
 *   else dMd + 2 alpha dMp + alpha^2 pMp >= Delta^2:  d += tau p, BOUNDARY;
 * d_H_d then gains tau^2 p^T (H + shift) p (d^T H p = 0 by conjugacy) and rel_residual is that of the iterate before the
 * boundary step.  With Delta_c = +inf every component's d and record is bitwise that of tsb_pcg_solve_ex, negative
 * curvature included (NEGCURV, NEGCURV_FIRST).  The solve's invariants hold: one writing kernel per field, no launch reads
 * what another CTA of it writes, no floating-point atomics, folds in a fixed order; check_every and the projected Hessian
 * (tsb_pcg_enable_psd) work as in tsb_pcg_solve_ex.
 * The first call on a workspace allocates the recurrence state, 32 bytes per component, with cudaMalloc;
 * tsb_pcg_device_bytes includes it from then on, and a workspace that never takes a trust-region solve keeps its size.
 * Make that first call outside any stream capture: on a stream being captured it returns TSB_E_INVALID, and a cudaMalloc
 * while another stream of the process is being captured in global mode invalidates that capture.
 * Argument errors (TSB_E_INVALID, nothing launched): those of tsb_pcg_solve_ex and a null radius_dev. */
int tsb_pcg_solve_tr(tsb_pcg_t s, const float *x_dev, const float *b_dev, const tsb_terms_t *terms,
                     const tsb_pcg_options_t *opt, const float *shift_dev, const float *radius_dev, float *d_out_dev,
                     tsb_pcg_sphere_t *spheres_out_dev, int32_t *iters_run_out, void *stream);

/* ---- Projected Hessian (projected Newton) ---------------------------------------------------------------------------
 * Opt-in on a solver workspace: every tet's Hessian in deformation-gradient space is replaced by its positive
 * semidefinite projection (same eigenvectors, negative eigenvalues clamped to 0), so the solve multiplies by
 *   H+(x) = c1 M + c2 sum_t K_t^T P(H_b,t) K_t + c3 sum_t K_t^T P(H_a,t) K_t       (K_t: dx -> dF = dDs Dm^-1)
 * which is PSD on every sphere: CG on it never stops at negative curvature from the tet terms, and a Levenberg-Marquardt
 * shift only has to regularise.  A tet is barrier-active where its det F < 0 and AMIPS-active where det F > 0 and
 * c3 != 0 (det F in fp64 from the fp32 positions: its sign can differ from the energy kernel's fp32 J only for |J| within
 * rounding of 0).  The projection uses the closed form of isotropic energies (signed SVD F = U diag(s) V^T, U and V proper
 * rotations; DESIGN.md section 5, "Projected Hessian").  This is a different model, not another implementation of the
 * exact one: iterates differ from the exact mode's, and the exact-mode calls are unchanged.
 *
 * tsb_pcg_enable_psd: rest_xyz (host float32 [3n]) and tets (host int32 [4 nele]) must be the mesh the workspace's handle
 * was created from.  Checks nele against the handle (TSB_E_INVALID), and every vertex id against [0, n) and every tet's
 * four vertices against the handle's components (TSB_E_MESH); computes Dm^-1 per tet in fp64 (stored as fp32; a zero-volume
 * rest tet is TSB_E_MESH), builds the per-vertex incidence lists of (tet, corner) ascending on the host, and allocates the
 * per-tet operators and the corner scratch.  After it, tsb_pcg_device_bytes has grown by
 *   237 nele + 4 (n + 1) + 16 ceil(nele / 256) + 16   bytes
 * (tet ids 16, Dm^-1 36, operator 120, activity 1, corner vectors 48 and incidence entries 16 per tet); the handle's
 * info.device_bytes is unchanged, and a workspace that never enables the mode keeps its size.  A second call is
 * TSB_E_INVALID.  After a failure the workspace is as before.
 * CAPTURE: the call is synchronous and allocates with cudaMalloc; it takes no stream, so it can only see a capture on the
 * legacy default stream (then TSB_E_INVALID).  A capture on any other stream is NOT detected: cudaMalloc then fails
 * (TSB_E_NOMEM with the CUDA message) and, in global capture mode, invalidates that capture.  Make the call before any
 * capture starts (DevicePCG(hessian="psd") refuses to run while torch's current stream is capturing).
 *
 * tsb_pcg_hvp_psd: projects at x, then hv_out = H+(x) v (device float32 [3n], fully overwritten, required) and
 *   curv_out = { c1 vMv + c2 vHb+v + c3 vHa+v, vMv, vHb+v, vHa+v }     (optional device float[4])
 * with vHb+v and vHa+v unweighted sums over the active tets.  c1, c2, order, c3 from *terms with tsb_hvp_ex's rules, and
 * c1, c2, c3 >= 0 (a negative or NaN coefficient is TSB_E_INVALID: the projection does not commute with a negative
 * weight).  Launches: the projection (one thread per tet), tsb_hvp_ex with c2 = c3 = 0 for c1 M v (its tet pass then adds
 * exact zeros), the tet kernel that writes each active tet's weighted corner vectors to the scratch, the vertex gather
 * that adds each vertex's active corners in incidence-list order (and, with curv_out, one fold kernel).
 *
 * With the mode enabled, tsb_pcg_solve(_ex) runs one projection launch before its loop and the projected product in place
 * of tsb_hvp_ex; the records' d_H_d is then d^T (H+ + mu I) d.  tsb_newton_step and tsb_newton_prox_step on a Newton
 * workspace over this solver workspace follow with no change of signature (their pred then models H+), and reject
 * negative coefficients.  The preconditioner stays the exact tsb_hess_diag blocks, clamped by tsb_pcg_set_blocks(_ex).
 * Invariants: no host read and no allocation after enable (everything is capturable in a CUDA graph); no floating-point
 * atomics in the new kernels and every per-vertex sum in incidence-list order, so hv, curv, d and the records are bitwise
 * identical across calls, streams and graph replays, on default and deterministic handles alike (the two give the same
 * bits for the same options), and a sphere's rows do not depend on another sphere's x or v.
 * Argument errors (nothing launched): a null workspace, x_dev, v_dev, terms or hv_out_dev, hv_out_dev equal to x_dev or
 * v_dev (hv is written before x and v are read for the last time; partial overlaps are the caller's to avoid), the mode not
 * enabled, an order other than 2 or 4, terms->c3 != 0 on a handle without enable_amips, a negative coefficient. */
int tsb_pcg_enable_psd(tsb_pcg_t s, const float *rest_xyz, const int32_t *tets, int32_t nele);
int tsb_pcg_hvp_psd(tsb_pcg_t s, const float *x_dev, const float *v_dev, const tsb_terms_t *terms, float *hv_out_dev,
                    float *curv_out_dev, void *stream);

/* ---- Assembled Hessian: the matrix a solver workspace multiplies by, as 3x3 block-CSR ------------------------------
 * A Hessian workspace sits beside a solver workspace (which must outlive it) and follows its mode at creation:
 *   exact:  H(x)  = c1 M + c2 sum_t K_t^T H_b,t K_t + c3 sum_t K_t^T H_a,t K_t
 *   PSD:    H+(x) with every tet block replaced by the projection tsb_pcg_hvp_psd applies (tsb_pcg_enable_psd first)
 * Layout: block rows over all n vertices, crow int32 [n + 1], col int32 [nnzb] (global vertex ids, ascending inside a
 * row), values float32 [nnzb][3][3] row-major, both triangles stored: torch.sparse_bsr_tensor(crow, col, values) and
 * scipy.sparse.bsr_matrix((values, col, crow)) take them as they are.  The pattern is M's off-diagonal pattern plus the
 * diagonal: every vertex some tet references has its diagonal block, an orphan vertex's row is empty, no block couples
 * two components.  Activity as in the PSD mode: barrier where det F < 0, AMIPS where det F > 0 and c3 != 0, det F in fp64
 * from the fp32 positions (its sign can differ from the energy kernel's fp32 J only for |J| within rounding of 0).
 *
 * tsb_hessian_create: rest_xyz (host float32 [3n]) and tets (host int32 [4 nele]) must be the mesh the handle was created
 * from (TSB_E_INVALID for another nele, TSB_E_MESH for a bad tet or other components).  Builds the block pattern on the
 * host (a mesh with 2^31 or more blocks is TSB_E_INVALID: shard it) and allocates, reported by tsb_hessian_device_bytes:
 *   8 (n + 1) + 8 nnzb + 493 nele   bytes (exact)          8 (n + 1) + 8 nnzb + 561 nele   bytes (PSD)
 * (row offsets and incidence offsets 4 (n + 1) each; columns and M weights 4 each per block; per tet: the 16 corner-pair
 * block indices 64, incidence entries 16, activity 1, the 10 weighted 3x3 blocks of its Hessian 360, and tet ids 16 plus
 * Dm^-1 36 (exact) or a private projection operator 120 (PSD, tet ids and Dm^-1 are the solver workspace's)).  Creating
 * one changes nothing about the handle or the solver workspace.  Synchronous, allocates: not during a stream capture
 * (detected on the legacy default stream only, as for tsb_pcg_enable_psd).
 *
 * tsb_hessian_pattern: *nnzb (optional) and, when non-null, copies crow (device int32 [n + 1]) and col (device int32
 * [nnzb]) on the stream.
 *
 * tsb_hessian_assemble: values_dev (device float32 [9 nnzb], fully overwritten) at x_dev (device float32 [3n]).  c1, c2,
 * order, c3 from *terms with tsb_hvp_ex's rules; in PSD mode c1, c2, c3 >= 0.  Launches: (PSD) the projection, the
 * per-tet block kernel, the row gather (c1 M_ij I plus the active tets' blocks of the row in incidence-list order).  No
 * host read, no allocation, no floating-point atomics: capturable in a CUDA graph, bitwise repeatable, equal on default,
 * deterministic and force_global handles of one mesh; blocks (i, j) and (j, i)^T are bitwise equal; a sphere's blocks do
 * not depend on another sphere's x.  Like the solver workspace it serves one stream at a time.
 * Argument errors (TSB_E_INVALID, nothing launched): a null workspace, x_dev, terms or values_dev, an order other than 2
 * or 4, terms->c3 != 0 on a handle without enable_amips, a negative coefficient in PSD mode. */
typedef struct tsb_hessian_s *tsb_hessian_t;
int tsb_hessian_create(tsb_pcg_t s, const float *rest_xyz, const int32_t *tets, int32_t nele, tsb_hessian_t *out);
void tsb_hessian_destroy(tsb_hessian_t hs);
const char *tsb_hessian_last_error(tsb_hessian_t hs);   /* hs may be NULL: last tsb_hessian_create failure */
int64_t tsb_hessian_device_bytes(tsb_hessian_t hs);
int tsb_hessian_pattern(tsb_hessian_t hs, int64_t *nnzb, int32_t *crow_dev_out, int32_t *col_dev_out, void *stream);
int tsb_hessian_assemble(tsb_hessian_t hs, const float *x_dev, const tsb_terms_t *terms, float *values_dev, void *stream);

/* ---- Symmetric Gauss-Seidel preconditioner: multicolour block SGS from the assembled Hessian ------------------------
 * Opt-in on a solver workspace, in place of block Jacobi.  Per component, with A the assembled matrix of hs (H, or H+ in
 * PSD mode), Dt^-1 the clamped inverse diagonal blocks tsb_pcg_set_blocks(_ex) computes, and L, U = L^T the strict lower
 * and upper block parts of A in a multicolour order (colours ascending; vertices that share a tet, or any other block of
 * the pattern, never share a colour):
 *   M^-1 = (Dt + U)^-1 Dt (Dt + L)^-1 = W^T Dt W,  W = (Dt + L)^-1
 * applied as a forward sweep, colour by colour, y_i = Dt_i^-1 (r_i - sum_{col j < col i} A_ij y_j), then a backward sweep,
 * colours in reverse, z_i = y_i - Dt_i^-1 sum_{col j > col i} A_ij z_j.  M^-1 is SPD wherever every Dt_i is, indefinite A
 * included, so CG, Steihaug-Toint and every Newton step keep their rules; a vertex with the zero inverse block gets z_i = 0
 * (it does not move, as with block Jacobi).  The symmetry rests on A_ij = A_ji^T bitwise, which the assembly guarantees.
 * DESIGN.md section 5, "Symmetric Gauss-Seidel preconditioner".
 *
 * tsb_pcg_enable_sgs: hs must have been created over s (TSB_E_INVALID otherwise) and must outlive every later call on s.
 * Colours every component greedily on the host (vertices ascending, smallest free colour: deterministic), builds each
 * row's lists of earlier-colour and later-colour blocks and the per-component colour schedule, and allocates the
 * workspace's own values buffer.  tsb_pcg_device_bytes grows by
 *   36 nnzb + 8 (nnzb - rows) + 12 rows + 8 + 8 (n_components + 1) + 4 (total colours + n_components) + 4 n   bytes
 * (values; the two block lists; list offsets and schedule; component and colour-table offsets; colour table; colours;
 * rows = vertices some tet references, total colours = the sum over components).  A component whose
 * vector does not fit one CTA's shared memory (12 bytes per vertex: about 19 k vertices on an H100) is TSB_E_INVALID,
 * naming the component and its size.  A second call is TSB_E_INVALID.  Synchronous and allocating: not during a stream
 * capture (detected on the legacy default stream only, as for tsb_pcg_enable_psd).  After a failure the workspace is as
 * before.  From then on every tsb_pcg_solve(_ex, _tr) on s applies M^-1 where block Jacobi applied its blocks (one sweep
 * kernel after the init and after every update kernel; the Jacobi z they write is overwritten), the trust-region
 * radius start of tsb_newton_tr_step(_ex) uses b^T M^-1 b, and every Newton step on s calls tsb_pcg_set_matrix in place
 * of tsb_hess_diag (the diagonal planes, and so the preconditioner and the first damping mu_c, then come from A).
 *
 * tsb_pcg_set_matrix: assembles A(x_dev) into the workspace's values buffer through hs (tsb_hessian_assemble's rules for
 * *terms) and writes its diagonal blocks to diag_out_dev (device float32 [2][n][3], tsb_hess_diag's planes; orphan rows
 * zero), to hand to tsb_pcg_set_blocks(_ex).  No host read, no allocation: capturable.
 *
 * tsb_pcg_apply_precond: z_dev = M^-1 r_dev on every component (device float32 [3n]; z on vertices no tet references is
 * left as it is; z_dev must not alias r_dev).  One launch, one CTA per component, no atomics: bitwise repeatable, and a
 * component's z does not depend on other components' r.
 *
 * tsb_pcg_sgs_colors: colors_out_dev (optional device int32 [n]) receives every vertex's colour (-1 for orphans), on the
 * legacy default stream and synchronously; *n_colors_out (optional) the most colours of any component.
 * Argument errors (TSB_E_INVALID, nothing launched): a null pointer that is required, SGS not enabled (set_matrix,
 * apply_precond, colors). */
int tsb_pcg_enable_sgs(tsb_pcg_t s, tsb_hessian_t hs);
int tsb_pcg_set_matrix(tsb_pcg_t s, const float *x_dev, const tsb_terms_t *terms, float *diag_out_dev, void *stream);
int tsb_pcg_apply_precond(tsb_pcg_t s, const float *r_dev, float *z_dev, void *stream);
int tsb_pcg_sgs_colors(tsb_pcg_t s, int32_t *colors_out_dev, int32_t *n_colors_out);

/* ---- Affine coarse space: a two-level preconditioner for the per-sphere solve --------------------------------------
 * Opt-in on a solver workspace, on top of block Jacobi or SGS (P below: the blocks, or the sweep's M^-1).  Per sphere c,
 * with Y_i = X_i - mean_c X (rest positions, the mean in fp64, Y stored in fp32) and the 9 coarse unknowns a 3 x 3 matrix
 * A, (Z a)_i = A Y_i spans the linear affine motions of the sphere, and the preconditioner is
 *   P + Z E+ Z^T,   E = E_c + shift_c (S_c (x) I3),   S_c = sum_i Y_i Y_i^T,
 * E_c = Z^T H Z = sum_t [c2 d2psi_b + c3 d2psi_a](F_t) (the c1 M term vanishes: M annihilates affine maps; translations
 * have no curvature), in PSD mode with the projected operator the solve multiplies by.  E+ is E's pseudo-inverse: cyclic
 * Jacobi in fp64, eigenvalues <= coarse_floor * lambda_max give 0, lambda_max <= 0 gives the zero matrix.  So the
 * preconditioner is SPD wherever P is, indefinite H included, and CG, Steihaug-Toint and every Newton rule keep their
 * meaning: with R = Z^T r, r.z becomes r.P r + R^T E+ R and z = P r + Z E+ R wherever the solve uses z (the first
 * direction, NEGCURV_FIRST's d, and tsb_pcg_solve_tr's norm).  It removes the near-null global modes
 * (rotations, scaling, shears with AMIPS or in PSD mode) that block Jacobi leaves to CG.  The R partials ride in the init
 * and update kernels and the fold in the direction kernel: no launch per iteration.  DESIGN.md section 5, "Affine coarse
 * space".
 *
 * tsb_pcg_enable_coarse: rest_xyz (host float32 [3n]) and tets (host int32 [4 nele]) must be the mesh the handle was
 * created from; coarse_floor >= 0.  Builds Y in the solver's vertex order, S_c, and per sphere a table of tet chunks of
 * <= 256 tets (tets grouped by sphere, ascending), and allocates, added to tsb_pcg_device_bytes:
 *   12 rows + 72 chunks + 372 tet_chunks + 700 n_components + 56 nele + 4   bytes
 * (Y; R partials; E_c partials and the chunk table; S_c, E+ and the chunk offsets; tet ids, vertices and Dm^-1 in chunk
 * order).  A workspace that never enables keeps its size.  E+ starts at 0 (no correction) until set_coarse.  Synchronous
 * and allocating: not during a stream capture (detected on the legacy default stream only, as for tsb_pcg_enable_psd).
 * A second call is TSB_E_INVALID; after a failure the workspace is as before.
 *
 * tsb_pcg_set_coarse: forms E_c at x_dev (tsb_hessian_assemble's rules for *terms; exact mode: barrier where det F < 0,
 * AMIPS where det F > 0 and c3 != 0, det F in fp64 from the fp32 x; PSD mode: runs the solve's projection launch first,
 * so the same x gives the same operator bits) and E+ of the unshifted E_c.  One thread per tet writes each tet chunk's
 * fp64 partials, summed in a fixed order; one thread per sphere folds them in chunk order and factors.
 * tsb_pcg_set_blocks(_ex) factors again with its shift, so the solve's E includes shift_c.  No host read, no
 * allocation, no atomics: capturable and bitwise repeatable; a sphere's E depends on its own x only.  Every damped or
 * proximal Newton step on a coarse workspace forms E_c after the diagonal blocks (or tsb_pcg_set_matrix) and leaves the
 * factorisation to its tsb_pcg_set_blocks_ex.  tsb_newton_tr_step(_ex) refuses a coarse workspace with TSB_E_INVALID:
 * the two-level norm is near-singular along the coarse modes, so the radius admits long affine moves that the gain
 * ratio rejects, and the steps stall (DESIGN.md section 5).
 *
 * tsb_pcg_coarse_matrix: E_out_dev (device double [n_components][81], component order) = the unshifted E_c of the last
 * set_coarse, on the legacy default stream and synchronously.
 *
 * tsb_pcg_apply_precond applies P + Z E+ Z^T at the current E+ on a coarse workspace (z on vertices no tet references is
 * left as it is).
 * Argument errors (TSB_E_INVALID, nothing launched): a null pointer that is required, coarse not enabled, a negative or
 * NaN coarse_floor, another nele, tets that do not match the handle's mesh (a vertex out of range, a tet across two of
 * its spheres, a zero-volume rest tet), the rules of *terms. */
int tsb_pcg_enable_coarse(tsb_pcg_t s, const float *rest_xyz, const int32_t *tets, int32_t nele, float coarse_floor);
int tsb_pcg_set_coarse(tsb_pcg_t s, const float *x_dev, const tsb_terms_t *terms, void *stream);
int tsb_pcg_coarse_matrix(tsb_pcg_t s, double *E_out_dev);

/* ---- Damped Newton step: one Levenberg-Marquardt iteration per sphere on the device (no counterpart in the reference)
 * A Newton workspace sits beside a solver workspace (which must outlive it; creating one changes nothing about the
 * handle or the solver workspace) and holds b, d and the two diagonal planes (12 floats per vertex), the per-sphere line
 * search outputs, the step-size table alpha_k = 2^-k (k < TSB_LINE_MAX_ALPHA), the per-sphere state (mu, nu, status,
 * whether mu is initialised), three fp64 partials per chunk and the per-sphere step sizes.  Device memory, reported by
 * tsb_newton_device_bytes:
 *   48 n + 24 chunks + 172 n_components + 176   bytes
 * (chunks as for tsb_pcg_device_bytes), plus 8 max(chunks, 1) bytes once a tsb_newton_prox_step (or a proximal
 * tsb_newton_tr_step) has been made and 20 n_components bytes once a tsb_newton_tr_step has been made.  A
 * new workspace is reset (every sphere ACTIVE, mu not initialised).  Like the handle and the solver workspace it serves
 * one stream at a time, and it shares the solver workspace's scratch. */
typedef struct tsb_newton_s *tsb_newton_t;
int tsb_newton_create(tsb_pcg_t s, tsb_newton_t *out);
void tsb_newton_destroy(tsb_newton_t nw);
const char *tsb_newton_last_error(tsb_newton_t nw);   /* nw may be NULL: last tsb_newton_create failure */
int64_t tsb_newton_device_bytes(tsb_newton_t nw);

/* Marks every sphere ACTIVE with mu not initialised (one memset on the stream; capturable); after a tsb_newton_tr_step
 * also the trust-region radius (a second memset), and after a tsb_newton_lbfgs_step every sphere's L-BFGS history is
 * emptied (another memset). */
int tsb_newton_reset(tsb_newton_t nw, void *stream);

enum {
  TSB_NEWTON_ACTIVE = 0,      /* still iterating                                                             */
  TSB_NEWTON_CONVERGED = 1,   /* |grad_c| <= gtol: frozen                                                     */
  TSB_NEWTON_STALLED = 2      /* no acceptable step with mu_c at mu_max: frozen                                */
};

typedef struct {            /* 64 bytes */
  int32_t max_iter;         /* >= 1: the damped solve enqueues exactly max_iter iterations (check_every = 0)        */
  float rtol;               /* >= 0: the solve's residual test                                                       */
  float rel_floor;          /* >= 0: the preconditioner's eigenvalue floor (tsb_pcg_set_blocks)                      */
  float tau;                /* > 0: initial mu_c = tau * max over the sphere's vertices of the diagonal entries D_ii  */
  float mu_min, mu_max;     /* 0 < mu_min <= mu_max, finite: bounds on mu_c                                          */
  float gtol;               /* >= 0: a sphere with |grad_c| <= gtol is CONVERGED                                     */
  float sigma;              /* in (0, 1): Armijo constant (1e-4 is the usual choice)                                 */
  float eta;                /* in (0, 1]: a step must lie below eta times the sphere's inversion-free step (0.9)      */
  int32_t n_alpha;          /* 1..TSB_LINE_MAX_ALPHA: step sizes 1, 1/2, ..., 2^-(n_alpha - 1)                       */
  int32_t reserved[6];      /* must be 0                                                                             */
} tsb_newton_options_t;

typedef struct {            /* one per component, component order of tsb_energy_grad_spheres; 64 bytes               */
  double mu;                /* mu_c after this step's update                                                         */
  double rho;               /* gain ratio of the full step, -dE_c(1) / pred (1 when pred <= 0); 0 when no decision ran */
  float grad_norm;          /* |grad_c| at x before the step (0 on a sphere already frozen: its right-hand side is 0) */
  float alpha;              /* the step taken (0: none)                                                              */
  float delta;              /* E_c(x + alpha d) - E_c(x) from the line search (0 if no step)                          */
  float b_dot_d;            /* b_c . d_c, b = -grad                                                                   */
  int32_t k;                /* index of the step size taken, -1 when none                                            */
  int32_t pcg_status;       /* TSB_PCG_* of the damped solve                                                         */
  int32_t n_hvp;            /* products in which the sphere was active in the solve                                  */
  int32_t status;           /* TSB_NEWTON_* after the step                                                           */
  int32_t first_vertex;     /* its lowest vertex id                                                                  */
  int32_t reserved[3];
} tsb_newton_sphere_t;

/* One damped Newton iteration on every sphere; x_dev (device float32 [3n]) is updated in place.  c1, c2, order, c3 from
 * *terms with tsb_hvp_ex's rules.  On one stream, without any host read (capturable in a CUDA graph), in this order:
 *   1. b = -grad E(x) (one gradient launch, gradH = -1); b_c = 0 on spheres already frozen, so their solve is ZERO_RHS;
 *   2. tsb_hess_diag;  3. on a sphere's first step, mu_c = tau * max_v max_i (D_v)_ii clamped to [mu_min, mu_max];
 *   4. tsb_pcg_set_blocks_ex and tsb_pcg_solve_ex with shift mu_c (fp32);  5. per sphere b.d and |d|^2 (fp64, fixed order);
 *   6. tsb_line_search at alpha_k = 2^-k, k < n_alpha, per sphere;  7. the decision below;  8. tsb_sphere_axpy in place.
 * Decision per sphere c, with g = |b_c| (from the solve's fp64 |b_c|^2), bd and dHd the solve's b.d and d^T (H + mu I) d
 * rounded to fp32 as tsb_pcg_sphere_t reports them, dd = |d_c|^2, dE_k = E_c(x + alpha_k d) - E_c(x) and alpha^ the
 * sphere's inversion-free step over (0, 1] (both from the line search):
 *   frozen: alpha = 0.  g <= gtol: CONVERGED, frozen, alpha = 0.
 *   k* = the smallest k with alpha_k < eta alpha^ and dE_k <= -sigma alpha_k bd; none (or bd <= 0): alpha = 0, k = -1.
 *   pred = bd - (dHd - mu' dd) / 2, mu' = the fp32 shift the solve used;  rho = -dE_0 / pred if pred > 0, else 1.
 *   k* = 0: mu = max(mu_min, mu max(1/3, 1 - (2 rho - 1)^3)), nu = 2;  otherwise mu = min(mu_max, mu nu), nu = 2 nu.
 *   no step and mu = mu_max: STALLED, frozen.      (mu, nu and rho in fp64)
 * records_out_dev (optional, device [info.n_components]) receives one tsb_newton_sphere_t per sphere.  No floating-point
 * atomics in the new kernels and every fold in a fixed order: on a deterministic handle x and the records are bitwise
 * identical across calls, streams and graph replays, and a sphere's trajectory does not depend on the other spheres.
 * Vertices no tet references never move.  Argument errors (TSB_E_INVALID, nothing launched): a null nw, x_dev, terms or
 * opt, an option outside its range above (NaN included), nonzero reserved words, an order other than 2 or 4,
 * terms->c3 != 0 on a handle without enable_amips.  DESIGN.md section 5, "Damped Newton step". */
int tsb_newton_step(tsb_newton_t nw, float *x_dev, const tsb_terms_t *terms, const tsb_newton_options_t *opt,
                    tsb_newton_sphere_t *records_out_dev, void *stream);

/* ---- Proximal Newton step: the geometry energy plus a per-sphere pull toward an anchor --------------------------
 * One damped Newton iteration, on every sphere c, of the proximal objective
 *   Phi_c(x) = E_c(x) + (w_c / 2) |x_c - y_c|^2        (summed over the vertices of c)
 * with E = c1 smooth + c2 barrier (+ c3 amips) from *terms as in tsb_newton_step.  anchor_dev: device float32 [3n], the
 * anchor y; weight_dev: device float32 [info.n_components], w_c in the component order of tsb_energy_grad_spheres.  Both
 * are read on the device, so a captured graph can be replayed after new anchor data and new weights are copied into the
 * same buffers.  The use: a first-order optimiser takes its step on the data term alone, giving y, and this call then
 * pulls the geometry energy down without moving far from y (the Hessian H + w_c I stays block diagonal by sphere).  A
 * linear term needs no separate support: q.x + (w/2)|x - x0|^2 = (w/2)|x - (x0 - q/w)|^2 + const, so a caller with a
 * linearised data gradient q passes the anchor x0 - q/w.
 *
 * tsb_newton_step's eight phases, options, records and invariants, with these changes:
 *   1. after the gradient launch, b_v += (-w_c)(x_v - y_v) on active spheres, each operation rounded on its own (no
 *      contraction), so that eager torch's b + (-w) * (x - y) gives the same bits; g = |b_c| = |grad Phi_c|, tested
 *      against gtol;
 *   3. on a sphere's first step mu_c = tau (max_v max_i (D_v)_ii + w_c), clamped as before; the solve's fp32 shift is
 *      fp32(mu_c + w_c), in tsb_pcg_set_blocks_ex and tsb_pcg_solve_ex alike (the record's mu is the damping alone);
 *   5. also d.(x - y) per sphere (fp64 partials per chunk, folded in a fixed order);
 *   7. the decision uses dPhi_k = dE_k + w_c (alpha_k d.(x - y) + alpha_k^2 |d|^2 / 2) (fp64) wherever the plain rule uses
 *      dE_k: in the Armijo test and in rho; pred = bd - (dHd - mu' dd) / 2 with mu' = double(shift) - double(w_c), since
 *      the solve's dHd is d^T (H + shift I) d; the inversion bound eta alpha^ is unchanged.
 * Records: the same layout; grad_norm is |grad Phi_c|, delta the dPhi of the step taken, b_dot_d uses b = -grad Phi.
 * A sphere whose w_c is NaN, infinite or negative gets b_c = 0 and alpha = 0 and is marked STALLED (frozen until
 * tsb_newton_reset): its vertices do not move.  With every w_c = 0 the call gives bitwise the x and records of
 * tsb_newton_step.  The new kernels use no floating-point atomics and fold in a fixed order, so the determinism and
 * independence statements of tsb_newton_step hold here too (a sphere's trajectory depends on its own anchor and weight
 * only).
 * The first call on a workspace allocates 8 max(chunks, 1) bytes for the d.(x - y) partials with cudaMalloc;
 * tsb_newton_device_bytes includes them from then on.  Make that first call outside any stream capture: on a stream
 * being captured it returns TSB_E_INVALID, and a cudaMalloc while another stream of the process is being captured in
 * global mode invalidates that capture.
 * Argument errors (TSB_E_INVALID, nothing launched): everything tsb_newton_step rejects, a null anchor_dev or
 * weight_dev, and anchor_dev == x_dev (x is updated in place while the anchor is read).  DESIGN.md section 5, "Proximal
 * Newton step". */
int tsb_newton_prox_step(tsb_newton_t nw, float *x_dev, const float *anchor_dev, const float *weight_dev,
                         const tsb_terms_t *terms, const tsb_newton_options_t *opt,
                         tsb_newton_sphere_t *records_out_dev, void *stream);

/* ---- Trust-region Newton step: one per-sphere trust-region iteration on the device ---------------------------------
 * Minimises E (anchor_dev = weight_dev = NULL) or the proximal objective Phi_c = E_c + (w_c / 2)|x_c - y_c|^2 (both set,
 * with tsb_newton_prox_step's semantics for the right-hand side, the d.(x - y) partials and an unusable weight) by a
 * trust-region step per sphere: no damping shift, but a radius Delta_c in the preconditioner norm inside which
 * tsb_pcg_solve_tr follows negative curvature to the boundary instead of stopping.  On one stream, without any host read
 * (capturable in a CUDA graph after the first call):
 *   1. b = -grad (prox: b -= w (x - y)); b_c = 0 on frozen spheres;  2. tsb_hess_diag;
 *   3. tsb_pcg_set_blocks_ex with shift w_c (prox) or none;
 *   4. on a sphere's first step after a reset, Delta_c = clamp(radius_init sqrt(b_c^T P b_c), radius_min, radius_max) (fp64);
 *   5. tsb_pcg_solve_tr with fp32(Delta_c) and shift w_c (prox) or none;  6. per sphere b.d and |d|^2 (and d.(x - y));
 *   7. tsb_line_search at the single step alpha = 1, per sphere;  8. the decision below;  9. tsb_sphere_axpy in place.
 * Decision per sphere c, in fp64, with g = |b_c|, bd and dHd the solve's b.d and d^T (H + w_c I) d rounded to fp32 as
 * tsb_pcg_sphere_t reports them, dMd = |d_c|_M^2 from the solve's recurrences, dPhi = Phi_c(x + d) - Phi_c(x) (dE for the
 * plain objective) and alpha^ the inversion-free step over (0, 1] from the line search:
 *   frozen: alpha = 0.  g <= gtol: CONVERGED, frozen.
 *   pred = bd - dHd / 2;  rho = -dPhi / pred if pred > 0, else 0 (the step is rejected).
 *   1 >= eta alpha^ (the full step would invert a tet): rejected, Delta = min(Delta / 4, eta alpha^ sqrt(dMd));
 *   else rho < 1/4 (or NaN): Delta = sqrt(dMd) / 4;  else rho > 3/4 on a BOUNDARY or NEGCURV_BOUNDARY solve:
 *   Delta = min(2 Delta, radius_max).
 *   accepted (alpha = 1) iff pred > 0, rho > accept and no tet inverts; rejected with Delta < radius_min: STALLED, frozen.
 * records_out_dev (optional, device [info.n_components]) receives one tsb_newton_tr_sphere_t per sphere.  No floating-point
 * atomics in the new kernels and every fold in a fixed order: on a deterministic handle x and the records are bitwise
 * identical across calls, streams and graph replays, and a sphere's trajectory depends on its own start, anchor and
 * weight only.  Vertices no tet references never move.
 * State: the radius and its init flag, 16 bytes per sphere, plus the fp32 radius, 4 bytes per sphere, allocated with the
 * solve's recurrence state (tsb_pcg_solve_tr) and, for the proximal objective, tsb_newton_prox_step's partials, by the
 * first call; tsb_newton_device_bytes grows by 20 n_components (+ 8 max(chunks, 1) if no proximal step was made yet) and
 * tsb_newton_reset re-arms the radius.  Make the first call outside any stream capture: on a stream being captured it
 * returns TSB_E_INVALID.
 * Argument errors (TSB_E_INVALID, nothing launched): a null nw, x_dev, terms or opt, exactly one of anchor_dev and
 * weight_dev null, anchor_dev == x_dev, an option outside its range (NaN included), nonzero reserved words, an order other
 * than 2 or 4, terms->c3 != 0 on a handle without enable_amips, a negative coefficient on a projected-Hessian workspace.
 * DESIGN.md section 5, "Trust-region Newton step". */
typedef struct {            /* 64 bytes */
  int32_t max_iter;         /* >= 1: the solve enqueues exactly max_iter iterations (check_every = 0)                   */
  float rtol;               /* >= 0: the solve's residual test                                                       */
  float rel_floor;          /* >= 0: the preconditioner's eigenvalue floor (tsb_pcg_set_blocks)                      */
  float gtol;               /* >= 0: a sphere with |grad_c| <= gtol is CONVERGED                                     */
  float radius_init;        /* > 0, finite: Delta_c = radius_init |b_c|_P on a first step, clamped                   */
  float radius_min;         /* 0 < radius_min <= radius_max < inf: a rejected step with Delta_c < radius_min STALLS  */
  float radius_max;
  float accept;             /* in [0, 1/4): a step is accepted when rho > accept (1e-4 is the usual choice)           */
  float eta;                /* in (0, 1]: the full step must lie below eta times the sphere's inversion-free step    */
  int32_t reserved[7];      /* must be 0                                                                             */
} tsb_newton_tr_options_t;

typedef struct {            /* one per component, component order of tsb_energy_grad_spheres; 64 bytes               */
  double radius;            /* Delta_c after this step's update                                                      */
  double rho;               /* -dPhi / pred (0 when pred <= 0 or no decision ran)                                    */
  float grad_norm;          /* |grad_c| at x before the step (0 on a sphere already frozen)                          */
  float alpha;              /* 1: the step was taken, 0: not                                                          */
  float delta;              /* Phi_c(x + d) - Phi_c(x) of the step taken (0 if none)                                 */
  float b_dot_d;            /* b_c . d_c, b = -grad                                                                   */
  float pred;               /* bd - dHd / 2, the model decrease (0 when no decision ran)                               */
  float d_norm;             /* |d_c|_M = sqrt(dMd)                                                                    */
  int32_t pcg_status;       /* TSB_PCG_* of the trust-region solve                                                    */
  int32_t n_hvp;            /* products in which the sphere was active in the solve                                  */
  int32_t status;           /* TSB_NEWTON_* after the step                                                           */
  int32_t first_vertex;     /* its lowest vertex id                                                                  */
  int32_t reserved[2];
} tsb_newton_tr_sphere_t;

int tsb_newton_tr_step(tsb_newton_t nw, float *x_dev, const float *anchor_dev, const float *weight_dev,
                       const tsb_terms_t *terms, const tsb_newton_tr_options_t *opt,
                       tsb_newton_tr_sphere_t *records_out_dev, void *stream);

/* ---- Backtracking trust-region Newton step: the trust-region step that takes a fraction of a rejected step ----------
 * tsb_newton_tr_step with bt == NULL (the same launches, the same bits).  With bt set, the same nine phases with two
 * changes: phase 7 runs tsb_line_search at the bt->n_alpha step sizes alpha_k = 2^-k of the workspace's table (as
 * tsb_newton_step does), and phase 8 is the rule below.  Per sphere, in fp64, with tsb_newton_tr_step's quantities
 * (pred, rho from dPhi_0 = dPhi at alpha = 1, eta alpha^, |d|_M) and dPhi_k = Phi_c(x + alpha_k d) - Phi_c(x):
 *   frozen, an unusable weight, g <= gtol: as tsb_newton_tr_step.
 *   the full step is accepted (no tet inverts, pred > 0, rho > accept): as tsb_newton_tr_step, radius update included.
 *   otherwise, if bd > 0, k* = the smallest k in [1, n_alpha) with alpha_k < eta alpha^ and
 *   dPhi_k <= -sigma alpha_k bd (the Armijo test of tsb_newton_step).  Found: the step alpha_{k*} d is taken and
 *   Delta = clamp(max(alpha_{k*} |d|_M, Delta / 4), radius_min, radius_max) (Delta before this step), so a step limited
 *   by the inversion bound alone shrinks the radius by at most the quarter of a poor model instead of down to
 *   eta alpha^ |d|_M.  Not found: rejected with tsb_newton_tr_step's radius update; then Delta < radius_min: STALLED.
 * Records: tsb_newton_tr_sphere_t; alpha is the fraction taken (1, 2^-k* or 0) and delta its dPhi.  No floating-point
 * atomics and every fold in a fixed order: the determinism and independence statements of tsb_newton_tr_step hold.  No
 * device memory beyond tsb_newton_tr_step's (the line search's per-sphere outputs are sized for TSB_LINE_MAX_ALPHA
 * steps from tsb_newton_create on); the first call allocates exactly as that one does and cannot be captured.
 * Argument errors (TSB_E_INVALID, nothing launched): everything tsb_newton_tr_step rejects, n_alpha outside
 * [2, TSB_LINE_MAX_ALPHA], sigma outside (0, 1/2) (NaN included), nonzero reserved words.  DESIGN.md section 5,
 * "Backtracking trust-region step". */
typedef struct {            /* 32 bytes */
  int32_t n_alpha;          /* 2..TSB_LINE_MAX_ALPHA: step sizes alpha_k = 2^-k, k < n_alpha                          */
  float sigma;              /* in (0, 1/2): the Armijo constant                                                        */
  int32_t reserved[6];      /* must be 0                                                                               */
} tsb_newton_backtrack_t;

int tsb_newton_tr_step_ex(tsb_newton_t nw, float *x_dev, const float *anchor_dev, const float *weight_dev,
                          const tsb_terms_t *terms, const tsb_newton_tr_options_t *opt, const tsb_newton_backtrack_t *bt,
                          tsb_newton_tr_sphere_t *records_out_dev, void *stream);

/* ---- L-BFGS step: per-sphere quasi-Newton steps from gradients and the line search, no Hessian products -----------
 * Minimises E (anchor_dev = weight_dev = NULL) or the proximal objective Phi_c = E_c + (w_c / 2)|x_c - y_c|^2 (both set,
 * with tsb_newton_prox_step's semantics for the right-hand side, the d.(x - y) term and an unusable weight) by one
 * limited-memory BFGS step per sphere.  Every sphere keeps its own history of up to m pairs (s_i, y_i) (the Hessian is
 * block diagonal by sphere), and the initial inverse Hessian is H0 = P, the block-Jacobi preconditioner a damped step
 * on this workspace builds with mu = 0, rebuilt at every step's x.  On one stream, without any host read (capturable in
 * a CUDA graph after the first call):
 *   1. b = -grad Phi(x) (one gradient launch, gradH = -1; b_c = 0 on frozen spheres and where w_c is unusable);
 *   2. tsb_hess_diag and tsb_pcg_set_blocks_ex with shift w_c (prox) or none: H0 = P;
 *   3. the direction kernel, one CTA per sphere, the history in global memory (no limit on a sphere's size):
 *      if the sphere moved on the previous step, s = x - x_prev (from a stored fp32 copy of x, so an x edited between
 *      calls is still right) and y = b_prev - b; the pair is kept, the oldest dropped from a full ring, when
 *      s.y > curv_eps |s| |y| (fp64);  the two-loop recursion with H0 = P, fp32 vectors and fp64 rho_i = 1 / s_i.y_i,
 *      alpha_i and dots;  if b.d <= 0 on a sphere with a history, the history is cleared and d = P b;  then x_prev, b_prev
 *      and the per-sphere b.b, b.d, |d|^2 (prox: d.(x - y)) in fp64;
 *   4. tsb_line_search at alpha_k = 2^-k, k < n_alpha, per sphere;  5. the decision below;  6. tsb_sphere_axpy in place.
 * Decision per sphere c, in fp64, with g = |b_c|, bd = b.d, dd = |d|^2, dPhi_k = dE_k + w_c (alpha_k d.(x - y) +
 * alpha_k^2 dd / 2) (dE_k for the plain objective; tsb_newton_prox_step's dPhi) and alpha^ the inversion-free step:
 *   frozen: alpha = 0.  An unusable w_c: STALLED, frozen.  g <= gtol: CONVERGED, frozen.
 *   k* = the smallest k with alpha_k < eta alpha^ and dPhi_k <= -sigma alpha_k bd (tsb_newton_step's Armijo test);
 *   none (or bd <= 0): no step, and the history is cleared; no step from an empty history (d = P b): STALLED, frozen.
 * records_out_dev (optional, device [info.n_components]) receives one tsb_newton_lbfgs_sphere_t per sphere.  No
 * floating-point atomics in the new kernels and every fold in a fixed order (one CTA owns a sphere: a fixed shuffle tree,
 * then the warps in order): on a deterministic handle x and the records are bitwise identical across calls, streams and
 * graph replays, and a sphere's trajectory depends on its own start, anchor and weight only.  Vertices no tet references
 * never move.  With every w_c = 0 the call gives bitwise the x and records of the call without an anchor.
 * State: the pairs (m + 1 slots of s and y per vertex: the slot being filled never holds a kept pair), x_prev, b_prev,
 * rho and a 64-byte record per sphere (ring head, count, whether it moved, the direction's dots), allocated by the first
 * call; tsb_newton_device_bytes grows by
 *   24 (m + 2) rows + 8 (m + 1) n_components + 64 n_components   bytes
 * (rows = vertices some tet references).  tsb_newton_reset empties every history (on a workspace that has one).  Make the
 * first call outside any stream capture: on a stream being captured it returns TSB_E_INVALID.  m is fixed by that call.
 * Argument errors (TSB_E_INVALID, nothing launched): a null nw, x_dev, terms or opt, exactly one of anchor_dev and
 * weight_dev null, anchor_dev == x_dev, an option outside its range (NaN included), nonzero reserved words, an m other
 * than the workspace's first one, an order other than 2 or 4, terms->c3 != 0 on a handle without enable_amips, a
 * negative coefficient on a projected-Hessian workspace, a workspace with the SGS preconditioner or the coarse space (H0
 * is block Jacobi only).  DESIGN.md section 5, "L-BFGS step". */
#define TSB_LBFGS_MAX_M 16
typedef struct {            /* 64 bytes */
  int32_t m;                /* 1..TSB_LBFGS_MAX_M: pairs kept per sphere; fixed by the workspace's first L-BFGS call    */
  float gtol;               /* >= 0: a sphere with |grad_c| <= gtol is CONVERGED                                     */
  float sigma;              /* in (0, 1): Armijo constant                                                            */
  float eta;                /* in (0, 1]: a step must lie below eta times the sphere's inversion-free step            */
  int32_t n_alpha;          /* 1..TSB_LINE_MAX_ALPHA: step sizes 1, 1/2, ..., 2^-(n_alpha - 1)                       */
  float rel_floor;          /* >= 0: H0's eigenvalue floor (tsb_pcg_set_blocks)                                      */
  float curv_eps;           /* >= 0, finite: a pair is kept only if s.y > curv_eps |s| |y| (fp64)                    */
  int32_t reserved[9];      /* must be 0                                                                             */
} tsb_newton_lbfgs_options_t;

typedef struct {            /* one per component, component order of tsb_energy_grad_spheres; 64 bytes               */
  float grad_norm;          /* |grad_c| at x before the step (0 on a sphere already frozen)                          */
  float alpha;              /* the step taken (0: none)                                                              */
  float delta;              /* Phi_c(x + alpha d) - Phi_c(x) of the step taken (0 if none)                            */
  float b_dot_d;            /* b_c . d_c, b = -grad                                                                   */
  float d_norm;             /* |d_c|                                                                                  */
  int32_t k;                /* index of the step size taken, -1 when none                                            */
  int32_t status;           /* TSB_NEWTON_* after the step                                                           */
  int32_t n_pairs;          /* pairs held after the step                                                             */
  int32_t pair_kept;        /* -1: no pair this step (the sphere did not move), 0: rejected by the curvature test, 1: kept */
  int32_t history_cleared;  /* 1: the history was cleared this step (b.d <= 0, or no step)                            */
  int32_t first_vertex;     /* its lowest vertex id                                                                  */
  int32_t reserved[5];
} tsb_newton_lbfgs_sphere_t;

int tsb_newton_lbfgs_step(tsb_newton_t nw, float *x_dev, const float *anchor_dev, const float *weight_dev,
                          const tsb_terms_t *terms, const tsb_newton_lbfgs_options_t *opt,
                          tsb_newton_lbfgs_sphere_t *records_out_dev, void *stream);

/* Same computation for callers whose vertex positions live in HOST memory (e.g. a CPU-side
 * optimiser): copies x_host -> device, runs the fused launch, copies energy[3] and grad back,
 * asynchronously; the outputs are valid once `stream` has been synchronised and the host buffers
 * must stay valid until then (pinned memory makes the copies truly asynchronous).  Calls
 * alternate between two internal streams (upload -> kernel -> download, each with its own staging buffers;
 * only the kernels are ordered across the two), so successive calls pipeline: call i+1's upload overlaps
 * call i's kernel and download.  Consequences: x_host must be fully
 * written by the CPU when the call is made (the upload is NOT ordered after earlier work queued on
 * `stream`), and the handle must not be used through tsb_energy_grad on another stream until `stream` has
 * been synchronised.  grad_out_host may be NULL.
 * Replaces the reference's implicit host round trips (the CPU scalar at tet_spheres_cuda.cu:194 and
 * the caller's .cpu() of the gradient). */
int tsb_energy_grad_host(tsb_handle_t h, const float *x_host, float c1, float c2, int32_t order,
                         float gradH, float *energy_out_host, float *grad_out_host, void *stream);

/* out = gradH * (*gradH_dev) * g  -- the cublasSscal at tet_spheres_cuda.cu:257-258 without the
 * .item() sync.  In-place allowed. */
int tsb_scale(const float *g_dev, int64_t count, float gradH, const float *gradH_dev,
              float *out_dev, void *stream);

/* Replaces tet_spheres_grad_limit (tet_spheres_cuda.cu:265-303) with what it was meant to do
 * (the reference reads grad[0] instead of the arg-max element and is unused by the trainer):
 * if max|grad| > s_threshold, grad *= s / max|grad|.  No host sync. */
/* work_dev: device float32 [4] scratch owned by the caller (zero-initialised once; the kernels leave
 * it zeroed), one per concurrently used stream -- like tsb_adam_uniform_step. */
int tsb_grad_limit(float *grad_dev, int64_t count, float s_threshold, float s, float *work_dev, void *stream);

/* "Next" row (f)1: AdamUniform.step (utils/optimizer.py:37-89) as two launches and no sync.
 * p, g1, g2: device float32 [count]; step is the 1-based step number AFTER increment.  lr and the
 * betas are doubles (Python floats) so that 1-beta and the bias corrections round as in the reference.
 * grad_limit <= 0 disables the clamp (optimizer.py:76-86).  work_dev: device float32 [4]
 * scratch owned by the caller (zero-initialised once; the kernels leave it zeroed). */
int tsb_adam_uniform_step(float *p_dev, const float *grad_dev, float *g1_dev, float *g2_dev,
                          int64_t count, double lr, double beta1, double beta2, int32_t step,
                          double grad_limit, float *work_dev, void *stream);

/* ---- "Next" row (f)2: surface gather + vertex-normal splat ------------------------------------------------
 * Replaces `tet_v[surface_vid]` (geometry/tetmesh_geometry.py:33) and `_compute_vertex_normal`
 * (geometry/tetmesh_geometry.py:39-66) and their autograd backward.  surface_vid: host int32 [nsv] tet-mesh
 * vertex of each surface vertex, each id at most once (a repeat is rejected with TSB_E_MESH: every gradient row has
 * one writer); surface_f: host int32 [3*nsf] triangles over surface-vertex ids.
 * One handle may serve one stream at a time (it owns a backward scratch array). */
typedef struct tsb_surface_s *tsb_surface_t;
int tsb_surface_create(const int32_t *surface_vid, int32_t nsv, const int32_t *surface_f, int32_t nsf,
                       int32_t n_tet_vertices, int device, tsb_surface_t *out);
void tsb_surface_destroy(tsb_surface_t s);
const char *tsb_surface_last_error(tsb_surface_t s);
/* v_pos_dev / v_nrm_dev: device float32 [3*nsv]; either may be NULL.  Normals: sum of cross(v1-v0, v2-v0) over the
 * incident faces in fixed order, (0,0,1) where |n|^2 <= 1e-20, then n / max(|n|, 1e-12). */
int tsb_surface_forward(tsb_surface_t s, const float *tet_v_dev, float *v_pos_dev, float *v_nrm_dev, void *stream);
/* grad_tet_v_dev: device float32 [3*n_tet_vertices], fully overwritten (zero for non-surface vertices);
 * grad_v_pos_dev / grad_v_nrm_dev: upstream gradients [3*nsv], either may be NULL. */
int tsb_surface_backward(tsb_surface_t s, const float *tet_v_dev, const float *grad_v_pos_dev,
                         const float *grad_v_nrm_dev, float *grad_tet_v_dev, void *stream);

/* ---- "Next" row (f)3: surface extraction on the GPU --------------------------------------------------------
 * Replaces get_surface_vf (geometry/mesh_utils.py:5-35; re-run by reset() / permute_surface_v(),
 * geometry/tetmesh_geometry.py:164-170,369-371) with identical output: the faces that belong to exactly one tet, in
 * lexicographic order of their sorted vertex triple, each in the orientation its tet gives it (face k opposite local
 * vertex k: (1,2,3), (0,3,2), (0,1,3), (0,2,1)), re-indexed into the increasing list of surface vertex ids.
 * tets_host: host int32 [4*nele], 0-based, entries in [0, n).  On success *surface_vid_out (int32 [*nsv_out]) and
 * *surface_f_out (int32 [3 * *nsf_out]) are host arrays owned by the caller: release them with tsb_free_host.
 * Synchronous (a setup call); errors are reported through tsb_setup_last_error (thread-local). */
int tsb_surface_extract(const int32_t *tets_host, int32_t nele, int32_t n, int device, int32_t *nsv_out,
                        int32_t *nsf_out, int32_t **surface_vid_out, int32_t **surface_f_out);
void tsb_free_host(void *p);
const char *tsb_setup_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* TSSPLAT_B200_H_ */
