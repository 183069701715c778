// Per-sphere L-BFGS step on the device (tsb_newton_lbfgs_step, include/tssplat_b200.h; DESIGN.md section 5, "L-BFGS
// step"): the direction kernel and the decision kernel.  The gradient, the preconditioner H0 = P, the line search and
// the step are the calls the damped Newton step makes.
//
// The direction kernel runs one CTA per sphere, which owns the whole sphere: every dot product is a per-thread sum over
// the thread's entries (entries e0 + t, e0 + t + kLT, ...), a shuffle tree and the warps in order (block_sum), so it
// needs no partial table, no second launch and no atomic, and a sphere's result does not depend on any other sphere.
// Every thread reads and writes only its own entries of the vectors, so the passes need no barrier beyond the sums'.
#include "tsb_device.cuh"
#include "tsb_lbfgs.cuh"

namespace tsb {
namespace {

constexpr int kLT = kLbfgsThreads;
constexpr int kDecideT = 256;        // decision kernel: thread = component

// Sum of v over the CTA in block_sum's fixed order, valid in every thread; sh holds kLT / 32 + 1 doubles.  The next
// call's first barrier comes after every thread has read the result, so sh can be reused at once.
__device__ __forceinline__ double cta_sum(double v, double *sh) {
  v = block_sum<kLT>(v, sh);
  if (threadIdx.x == 0) sh[kLT / 32] = v;
  __syncthreads();
  return sh[kLT / 32];
}

// q + a v per entry in fp64, rounded to fp32
__device__ __forceinline__ F3 axpy3(F3 q, double a, F3 v) {
  return F3{float(double(q.x) + a * double(v.x)), float(double(q.y) + a * double(v.y)), float(double(q.z) + a * double(v.z))};
}

// The direction of one sphere (CTA = component); see tsb_newton_lbfgs_step in the header.  Pair slots are indexed by
// the entry e of the component vertex list, the vectors b, d and x by the vertex id v = vert[e].
template <bool PROX>
__global__ void __launch_bounds__(kLT) lbfgs_dir_kernel(const PcgParams s, const NewtonParams w, const LbfgsParams l,
                                                        const LbfgsRule r, const float *__restrict__ x, const ProxParams p) {
  __shared__ double sh[kLT / 32 + 1];
  __shared__ double rho[TSB_LBFGS_MAX_M + 1], al[TSB_LBFGS_MAX_M];
  const int c = blockIdx.x, t = int(threadIdx.x);
  const int e0 = s.chunk[3 * s.comp_chunk[c] + 1], e1 = s.chunk[3 * (s.comp_chunk[c + 1] - 1) + 2];
  const int M1 = l.m + 1;
  const size_t slot = 3 * size_t(l.rows);          // floats per pair slot
  LbfgsComp L = l.comp[c];
  L.pair = -1;
  L.cleared = 0;
  bool live = w.comp[c].status == TSB_NEWTON_ACTIVE;
  if (PROX) live = live && prox_weight_ok(p.weight[c]);
  if (!live) {        // b_c = 0 and d_c = 0 (P b would be NaN where w_c is unusable); the history stays as it is
    for (int e = e0 + t; e < e1; e += kLT) st3(w.d, s.vert[e], F3{0.f, 0.f, 0.f});
    if (t == 0) {
      L.bb = L.bd = L.dd = L.dx = 0.0;
      l.comp[c] = L;
    }
    return;
  }
  if (t < M1) rho[t] = l.rho[size_t(c) * M1 + t];

  // The last step's pair into slot head, which never holds a kept pair (m + 1 slots for m pairs), so a rejected pair
  // costs nothing; x_prev = x, b_prev = b; q = b in d.
  float *sn = l.s + slot * L.head, *yn = l.y + slot * L.head;
  double bb = 0.0, sy = 0.0, ss = 0.0, yy = 0.0;
  for (int e = e0 + t; e < e1; e += kLT) {
    const int v = s.vert[e];
    const F3 xv = ld3(x, v), bv = ld3(w.b, v);
    if (L.moved) {
      const F3 xp = ld3(l.x_prev, e), bp = ld3(l.b_prev, e);
      const F3 sv{xv.x - xp.x, xv.y - xp.y, xv.z - xp.z}, yv{bp.x - bv.x, bp.y - bv.y, bp.z - bv.z};
      st3(sn, e, sv);
      st3(yn, e, yv);
      sy += dot3(sv, yv);
      ss += dot3(sv, sv);
      yy += dot3(yv, yv);
    }
    st3(l.x_prev, e, xv);
    st3(l.b_prev, e, bv);
    st3(w.d, v, bv);
    bb += dot3(bv, bv);
  }
  bb = cta_sum(bb, sh);
  if (L.moved) {
    sy = cta_sum(sy, sh);
    ss = cta_sum(ss, sh);
    yy = cta_sum(yy, sh);
    L.pair = sy > double(r.curv_eps) * sqrt(ss) * sqrt(yy) ? 1 : 0;
    if (L.pair) {
      if (t == 0) rho[L.head] = l.rho[size_t(c) * M1 + L.head] = 1.0 / sy;
      L.head = (L.head + 1) % M1;
      L.count = min(L.count + 1, l.m);
    }
  }
  __syncthreads();    // rho

  const int n = L.count;
  auto at = [&](int j) { return (L.head - 1 - j + 2 * M1) % M1; };   // slot of the j-th newest pair
  double bd = 0.0, dd = 0.0, dx = 0.0;
  auto dots = [&](int v, F3 z) {
    bd += dot3(ld3(w.b, v), z);
    dd += dot3(z, z);
    if (PROX) {
      const F3 xv = ld3(p.x, v), y = ld3(p.anchor, v);
      dx += double(z.x) * (double(xv.x) - double(y.x)) + double(z.y) * (double(xv.y) - double(y.y)) +
            double(z.z) * (double(xv.z) - double(y.z));
    }
  };

  // First loop, newest to oldest: alpha_j = rho_j s_j.q, q -= alpha_j y_j (each update applied in the next pass).
  double a = 0.0;
  const float *u = nullptr;
  for (int j = 0; j < n; ++j) {
    const float *sj = l.s + slot * at(j);
    double sq = 0.0;
    for (int e = e0 + t; e < e1; e += kLT) {
      const int v = s.vert[e];
      F3 q = ld3(w.d, v);
      if (u) {
        q = axpy3(q, -a, ld3(u, e));
        st3(w.d, v, q);
      }
      sq += dot3(ld3(sj, e), q);
    }
    a = rho[at(j)] * cta_sum(sq, sh);
    if (t == 0) al[j] = a;
    u = l.y + slot * at(j);
  }
  // r = H0 q = P q, with y_oldest.r for the second loop (or the dots when there is no pair)
  double yr = 0.0;
  {
    const float *yj = n ? l.y + slot * at(n - 1) : nullptr;
    for (int e = e0 + t; e < e1; e += kLT) {
      const int v = s.vert[e];
      F3 q = ld3(w.d, v);
      if (u) q = axpy3(q, -a, ld3(u, e));
      const F3 z = apply_block(s.pinv, v, q);
      st3(w.d, v, z);
      if (yj) yr += dot3(ld3(yj, e), z);
      else dots(v, z);
    }
    if (n) yr = cta_sum(yr, sh);
  }
  // Second loop, oldest to newest: beta_j = rho_j y_j.r, r += (alpha_j - beta_j) s_j; the last pass forms the dots.
  for (int j = n - 1; j >= 0; --j) {
    const double cf = al[j] - rho[at(j)] * yr;
    const float *sj = l.s + slot * at(j), *yj = j ? l.y + slot * at(j - 1) : nullptr;
    yr = 0.0;
    for (int e = e0 + t; e < e1; e += kLT) {
      const int v = s.vert[e];
      const F3 z = axpy3(ld3(w.d, v), cf, ld3(sj, e));
      st3(w.d, v, z);
      if (yj) yr += dot3(ld3(yj, e), z);
      else dots(v, z);
    }
    if (j) yr = cta_sum(yr, sh);
  }
  bd = cta_sum(bd, sh);
  dd = cta_sum(dd, sh);
  if (PROX) dx = cta_sum(dx, sh);
  if (!(bd > 0.0) && n > 0) {         // not a descent direction: clear the history, d = P b
    L.count = 0;
    L.cleared = 1;
    bd = dd = dx = 0.0;
    for (int e = e0 + t; e < e1; e += kLT) {
      const int v = s.vert[e];
      const F3 z = apply_block(s.pinv, v, ld3(w.b, v));
      st3(w.d, v, z);
      dots(v, z);
    }
    bd = cta_sum(bd, sh);
    dd = cta_sum(dd, sh);
    if (PROX) dx = cta_sum(dx, sh);
  }
  if (t == 0) {
    L.bb = bb;
    L.bd = bd;
    L.dd = dd;
    L.dx = dx;
    l.comp[c] = L;
  }
}

// Step choice, history clearing and records of every component (thread = component); see tsb_newton_lbfgs_step in the
// header.
template <bool PROX>
__global__ void __launch_bounds__(kDecideT) lbfgs_decide_kernel(const PcgParams s, const NewtonParams w, const LbfgsParams l,
                                                                const LbfgsRule r, tsb_newton_lbfgs_sphere_t *__restrict__ out,
                                                                const ProxParams p) {
  const int c = blockIdx.x * kDecideT + int(threadIdx.x);
  if (c >= s.n_components) return;
  NewtonComp N = w.comp[c];
  LbfgsComp L = l.comp[c];
  double wc = 0.0;
  bool bad_w = false;
  if (PROX) {
    const float q = p.weight[c];
    bad_w = !prox_weight_ok(q);
    wc = bad_w ? 0.0 : double(q);
  }
  const double g = sqrt(L.bb);
  int ks = -1;
  float alpha = 0.f, delta = 0.f;
  if (N.status == TSB_NEWTON_ACTIVE) {
    if (PROX && bad_w) {
      N.status = TSB_NEWTON_STALLED;
    } else if (g <= double(r.gtol)) {
      N.status = TSB_NEWTON_CONVERGED;
    } else {
      const float *dl = w.sphere_delta + size_t(c) * size_t(r.n_alpha) * 4;
      const double lim = double(r.eta) * double(w.sphere_step[c]);
      if (L.bd > 0.0)
        for (int k = 0; k < r.n_alpha; ++k) {
          const double a = double(w.alphas[k]);
          if (a < lim && step_change<PROX>(dl[4 * k], wc, a, L.dx, L.dd) <= -double(r.sigma) * a * L.bd) { ks = k; break; }
        }
      if (ks >= 0) {
        alpha = w.alphas[ks];
        delta = PROX ? float(step_change<PROX>(dl[4 * ks], wc, double(alpha), L.dx, L.dd)) : dl[4 * ks];
      } else if (L.count == 0) {        // no step along P b either
        N.status = TSB_NEWTON_STALLED;
      } else {
        L.count = 0;
        L.cleared = 1;
      }
    }
  }
  L.moved = alpha > 0.f;
  w.alpha_sphere[c] = alpha;
  w.comp[c] = N;
  l.comp[c] = L;
  if (!out) return;
  tsb_newton_lbfgs_sphere_t o;
  o.grad_norm = float(g);
  o.alpha = alpha;
  o.delta = delta;
  o.b_dot_d = float(L.bd);
  o.d_norm = float(sqrt(L.dd));
  o.k = ks;
  o.status = N.status;
  o.n_pairs = L.count;
  o.pair_kept = L.pair;
  o.history_cleared = L.cleared;
  o.first_vertex = s.vert[s.chunk[3 * size_t(s.comp_chunk[c]) + 1]];
  for (int k = 0; k < 5; ++k) o.reserved[k] = 0;
  out[c] = o;
}

}  // namespace

cudaError_t launch_lbfgs_dir(const PcgParams &s, const NewtonParams &w, const LbfgsParams &l, const LbfgsRule &r,
                             const float *x, const ProxParams *p, cudaStream_t st) {
  (p ? lbfgs_dir_kernel<true> : lbfgs_dir_kernel<false>)<<<unsigned(s.n_components), kLT, 0, st>>>(s, w, l, r, x,
                                                                                                     p ? *p : ProxParams{});
  return cudaGetLastError();
}

cudaError_t launch_lbfgs_decide(const PcgParams &s, const NewtonParams &w, const LbfgsParams &l, const LbfgsRule &r,
                                const ProxParams *p, tsb_newton_lbfgs_sphere_t *out, cudaStream_t st) {
  (p ? lbfgs_decide_kernel<true> : lbfgs_decide_kernel<false>)<<<unsigned((s.n_components + kDecideT - 1) / kDecideT),
                                                                  kDecideT, 0, st>>>(s, w, l, r, out, p ? *p : ProxParams{});
  return cudaGetLastError();
}

}  // namespace tsb
