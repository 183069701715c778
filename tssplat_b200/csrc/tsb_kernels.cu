// Fused geometry-energy + gradient kernel for sm_90a (H100), plus the small level-1 helpers.
//
// ONE launch replaces the reference's forward+backward pipeline
// (tssplat_ext/tet_spheres/tet_spheres_cuda.cu:118-263: SpMV GTLTLG.x, Sdot, SpMV G.x,
// cuda_forward_det, Sasum, SpMV c1.GTLTLG.x, SpMV G.x again, cuda_backward_det, SpMV G^T, Sscal,
// with three host syncs).
//
// Math (DESIGN.md section 3).  With u = x - X (X = rest positions; staged as u - u_r per component, in fp64):
//   smoothness  1/2 x^T M x = 1/2 u^T M u        M = G^T L^T L G  (tet_spheres.cpp:148; M X = 0: affine maps are in its null space)
//   M has zero row sums, so with d_ij = u_j - u_i
//       (M u)_i        = sum_{j != i} M_ij d_ij
//       1/2 u^T M u    = -1/4 sum_i sum_{j != i} M_ij |d_ij|^2
//   which is what each lane evaluates for its vertex row: well conditioned near the rest state
//   (the reference's fp32 x^T M x cancels there) and no scatter -- every gradient row has one writer.
//   barrier     sum_t max(-J_t, 0)^p,  J_t = det F_t = det(Ds_t) / det(Dm_t)   (cu:48-66; F = Ds Dm^-1)
//       dJ/dx_k = cof(Ds)[:,k] / det(Dm)  (k = 1..3),  dJ/dx_0 = -(sum)           (cu:68-102, :32-46)
//   so a tet needs 4 vertex ids + one float; only inverted tets (rare) touch the gradient, with
//   red.global.add.f32 after the component's rows have been stored (per-component counter).
//
// Execution.  Persistent CTAs (1 per SM x 16 warps, or 2 x 8).  Every warp owns a private byte
// stream of operator rows and tet blocks (tsb_plan.h) and pulls it through a private shared-memory
// ring with TMA bulk copies (cp.async.bulk + mbarrier complete_tx), issued by its lane 0: the first
// chunk before griddepcontrol.wait (plan data streams from HBM while the previous kernel drains), the rest of the
// ring once the loads of x have been issued, so that x does not queue behind them.
// Per segment the CTA stages u and x of the whole component in shared memory (float4 each; the next
// component is prefetched through registers), so all gathers are LDS.128.  Energies: per-lane fp64
// partials -> per-CTA pair -> last-arriving CTA folds them in fixed order (deterministic).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <utility>

#include "tsb_kernels.cuh"

namespace tsb {

namespace {

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// LINE's reduce-scatter of N (8 or 16) per-lane values: the halving with xor offset o = 16, 8, ... leaves the lanes with
// bit o set the upper half (h = N/2, N/4, ...), so value j ends in the lanes whose bits o are the bits h of j
template <int N>
__device__ __forceinline__ int line_lane(int j) {
  int l = 0;
#pragma unroll
  for (int h = N / 2, o = 16; h >= 1; h >>= 1, o >>= 1) l |= (j & h) ? o : 0;
  return l;
}

// ---- mbarrier + TMA bulk copy (1-D) ------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ unsigned int ld_acquire(const unsigned int *p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

constexpr int align_up(int v, int a) { return (v + a - 1) / a * a; }
constexpr int kMaxSlots = 8;
constexpr unsigned long long kSentinel = kEnergySentinel;   // "no partial yet" marker in cta_energy (a NaN payload)

// Profiling build only (-DTSB_TRACE, tools/trace_phases.py): thread 0 of every CTA stamps its phases in slots 0..15 of
// the CTA's kTraceSlots, lane 0 of warp w the return of its last chunk wait in slot 16 + w.
#ifdef TSB_TRACE
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define TSB_STAMP(i) do { if (tid == 0 && p.trace) p.trace[blockIdx.x * kTraceSlots + (i)] = (i) == 0 ? gtime() : (unsigned long long)clock64(); } while (0)
#else
#define TSB_STAMP(i) do { } while (0)
#endif

// shared-memory layout: staging area (offset 0: gather offsets in the plan are relative to it) | rings |
// mbarriers | fp64 reduction scratch
__host__ __device__ constexpr int off_rings(int stage_bytes) { return align_up(stage_bytes, 128); }
__host__ __device__ constexpr int off_bars(int stage_bytes, int nw, int ring) { return off_rings(stage_bytes) + nw * ring; }
__host__ __device__ constexpr int off_red(int stage_bytes, int nw, int ring) { return off_bars(stage_bytes, nw, ring) + nw * kMaxSlots * 8; }
constexpr int kSegTab = 16;   // segment headers (and per-warp block counts) of a CTA cached in shared memory; beyond that: global
__host__ __device__ constexpr int off_segtab(int stage_bytes, int nw, int ring) { return align_up(off_red(stage_bytes, nw, ring) + nw * 24, 32); }
__host__ __device__ constexpr int off_wsegtab(int stage_bytes, int nw, int ring) { return off_segtab(stage_bytes, nw, ring) + kSegTab * 32; }
__host__ __device__ constexpr int smem_total(int stage_bytes, int nw, int ring) { return align_up(off_wsegtab(stage_bytes, nw, ring) + kSegTab * nw * 4, 128); }

// ---- fp32 pairs: even and odd entries of a row accumulate in two independent FFMA chains -------------------
// (sm_90 has no packed fp32 FMA; two chains keep the latency of each dependent FMA off the critical path, and
// the rounding is that of the pairwise form: lo + hi at the row end)
struct f32x2 { float lo, hi; };
__device__ __forceinline__ f32x2 pk2(float lo, float hi) { return f32x2{lo, hi}; }
__device__ __forceinline__ float sum2(f32x2 v) { return v.lo + v.hi; }
__device__ __forceinline__ void fma2_acc(f32x2 &acc, f32x2 a, f32x2 b) { acc.lo = fmaf(a.lo, b.lo, acc.lo); acc.hi = fmaf(a.hi, b.hi, acc.hi); }

// Staged displacement of a vertex whose component is shifted by c (any value shared by the component: the operator's
// differences and the energy do not see it; the kernel takes c = u of the component's reference vertex):
// (x - X) - c to within about one rounding of the exact value.  x - X is kept exactly as s + e (TwoSum); when the
// component has moved far from rest, s and c are close and s - c is exact (Sterbenz), so the rigid displacement never
// enters a rounded difference.  At rest (x = X, c = 0) the result is exactly 0.
__device__ __forceinline__ float rel_u(float x, float X, float c) {
  const float s = x - X, bb = s - x;
  const float e = (x - (s - bb)) + (-X - bb);
  return (s - c) + e;
}

template <bool GLOBAL> struct Fmt;
template <> struct Fmt<false> { static constexpr uint32_t CELL = kCellStaged, IB = 2, TPL = 2; };   // 16-bit smem byte offsets
template <> struct Fmt<true> { static constexpr uint32_t CELL = kCellGlobal, IB = 4, TPL = 1; };    // 32-bit vertex ids

// Per-warp view of its TMA-fed cell stream: `cpc` cells per chunk, one chunk per ring slot, `nslot` slots.
// Lane 0 keeps the producer state (next source address, bytes left to request).
template <uint32_t CELL>
struct WarpStream {
  const unsigned char *next_src;   // lane 0: global address of the next chunk to request
  uint32_t bytes_left;             // lane 0: bytes of the stream not yet requested
  uint32_t bars;                   // shared-space address of this warp's mbarriers
  unsigned char *ring;             // this warp's ring
  unsigned char *cell;             // current cell
  uint32_t chunk_bytes, cpc, nslot;
  uint32_t cc, slot, phase, cells_left;
  int lane;
#ifdef TSB_TRACE
  unsigned long long *trace_last;  // lane 0: clock64 when the warp's latest chunk wait returned
#endif

  __device__ __forceinline__ void request(uint32_t smem_dst, uint32_t bar) {   // lane 0 only
    const uint32_t bytes = min(chunk_bytes, bytes_left);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst), "l"(next_src),
                 "r"(bytes), "r"(bar)
                 : "memory");
    next_src += bytes;
    bytes_left -= bytes;
  }
  __device__ __forceinline__ void wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
      asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
  }
  // Lane 0 requests the chunk of slot 0 before griddepcontrol.wait and those of the other slots here, once the CTA's
  // x loads have been issued: with the plan HBM-cold, the loads that stage x would otherwise queue behind every
  // warp's whole ring of plan data, although the warp needs only its first chunk before the staged x.
  __device__ __forceinline__ void request_rest() {
    if (lane == 0)
      for (uint32_t i = 1; i < nslot && bytes_left; ++i) request(smem_u32(ring) + i * chunk_bytes, bars + i * 8);
  }
  __device__ __forceinline__ void begin() {       // first chunk has landed
    if (cells_left) wait(bars, 0);
  }
  // cells of the current chunk not yet consumed (the caller may read up to that many cells from `cell` on)
  __device__ __forceinline__ uint32_t avail() const { return cpc - cc; }
  // n <= avail() cells starting at `cell` have been read into registers
  __device__ __forceinline__ void advance(uint32_t n) {
    cell += n * CELL;
    cc += n;
    cells_left -= n;
    if (cc == cpc) {                 // leave the chunk: refill its slot, wait for the next chunk
      cc = 0;
      __syncwarp();
      if (lane == 0 && bytes_left) request(smem_u32(cell) - chunk_bytes, bars + slot * 8);
      if (++slot == nslot) { slot = 0; cell = ring; phase ^= 1u; }
      if (cells_left) wait(bars + slot * 8, phase);
#ifdef TSB_TRACE
      if (cells_left && trace_last) *trace_last = (unsigned long long)clock64();
#endif
    }
  }
};

// DET (deterministic gradient, tsb_options_t.deterministic): a contributing tet stores its four corner vectors at its
// tet slot instead of adding them to grad, every tet cell stores its activity ballot, and the component is flagged;
// det_gather_kernel then adds them in a fixed order.  Tets never touch grad, so there is no rows-done protocol.
// SPH (tsb_energy_grad_spheres): at the end of every segment each warp reduces its lanes' energy partials, inverted-tet
// count and smallest J, and lane 0 stores them as the (segment, warp) record; the running totals move to the warp's
// red[] slot, so the CTA fold below is unchanged.  sphere_fold_kernel turns the records into per-component statistics.
// HVP (tsb_hvp, tsb_hvp_ex; never with SPH): the u slots hold v - v_ref instead of x - X, so the row pass yields M v, an
// inverted tet adds its H_t v instead of its gradient (through the same scratch or atomics), and the energy partials
// carry v^T M v and v^T H_t v (DESIGN.md section 5).  x stays in the x slots: the active set is the gradient's.  With
// AMIPS (and c3 != 0) a tet with J > 0 adds its H_a v the same way, and the AMIPS partial carries v^T H_a v.
// LINE (tsb_line_search; with AMIPS only): staged as HVP with v = d, so the row pass yields M d; a row adds d^T M d and
// u^T M d, every real tet its barrier (and AMIPS) change at each alpha_k and the first root of its det F along d.  No
// gradient, no energy fold: the CTA's warps combine their sums per segment into one LineRec (DESIGN.md section 5).
// DIAG (tsb_hess_diag; with AMIPS and DET only): staged as the gradient.  A row stores s1 M_ii = -s1 sum_j M_ij (its
// streamed weights, no gather), an inverted tet (and with AMIPS a tet with J > 0) the diagonal 3x3 blocks of its Hessian
// at its four corners, through the same scratch or atomics as the gradient (DESIGN.md section 5, "Hessian diagonal").
template <int NW, int MINB, bool GLOBAL, bool AMIPS, bool DET = false, bool SPH = false, bool HVP = false, bool LINE = false,
          bool DIAG = false>
__global__ void __launch_bounds__(NW * 32, MINB) energy_grad_kernel(const KParams p) {
  using F = Fmt<GLOBAL>;
  constexpr bool VS = HVP || LINE;   // the u slots hold a direction (v, or d) instead of x - X
  constexpr int NT = NW * 32;
  constexpr uint32_t CELL = F::CELL, WOFF = 128 * F::IB;
  constexpr int SV = GLOBAL ? 1 : (1024 + NT - 1) / NT;   // register-prefetch slots per thread (vh <= 1023)
  extern __shared__ __align__(128) unsigned char smem[];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ring = p.ring_bytes, stage_bytes = p.stage_bytes;
  TSB_STAMP(0); TSB_STAMP(1);
  double *red = reinterpret_cast<double *>(smem + off_red(stage_bytes, NW, ring));
  float4 *stage = reinterpret_cast<float4 *>(smem);

  // ---- prologue: plan data only (overlaps the previous kernel under programmatic dependent launch)
  const int2 cs = __ldg(&p.cta_seg[blockIdx.x]);
  WarpStream<CELL> ws;
  {
    const uint2 wd = __ldg(&p.wdesc[blockIdx.x * NW + warp]);
    ws.next_src = p.stream + size_t(wd.x) * 16;
    ws.bytes_left = wd.y;
    ws.cells_left = wd.y / CELL;
    ws.ring = smem + off_rings(stage_bytes) + warp * ring;
    ws.bars = smem_u32(smem + off_bars(stage_bytes, NW, ring)) + warp * kMaxSlots * 8;
    ws.cpc = uint32_t(p.cells_per_chunk);
    ws.chunk_bytes = ws.cpc * CELL;
    ws.nslot = uint32_t(p.ring_slots);
#ifdef TSB_TRACE
    ws.trace_last = (lane == 0 && p.trace) ? p.trace + blockIdx.x * kTraceSlots + 16 + warp : nullptr;
#endif
    ws.cell = ws.ring;
    ws.cc = 0; ws.slot = 0; ws.phase = 0; ws.lane = lane;
    if (lane == 0) {
      for (uint32_t i = 0; i < ws.nslot; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(ws.bars + i * 8), "r"(1) : "memory");
      mbar_fence_init();
      if (ws.bytes_left) ws.request(smem_u32(ws.ring), ws.bars);   // slot 0; the others: request_rest()
    }
    __syncwarp();
  }
  const int vh = p.vh;
  // float4 index of a segment's u / x arrays inside the staging area (must match tsb_plan.cpp)
  auto ubase_of = [&](const SegHdr &h, int li) -> int { return h.whole ? 0 : (li & 1) * 2 * vh; };
  auto xbase_of = [&](const SegHdr &h, int li) -> int { return h.whole ? h.npos : (li & 1) * 2 * vh + vh; };
  // global id of a segment's local vertex v
  auto gid_of = [&](const SegHdr &h, int v) -> size_t { return size_t(h.vbase >= 0 ? h.vbase + v : __ldg(&p.vlist[h.x4off + v])); };
  auto load_rest = [&](const SegHdr &h, float4 (&X)[SV]) {   // rest positions (.w: staging position) -> registers
#pragma unroll
    for (int k = 0; k < SV; ++k) {
      const int v = tid + k * NT;
      // HVP: load_x fills xyz with v, and store_staged_ref reads the staging position itself (register budget)
      if (!VS && v < h.nv) { X[k] = __ldg(&p.X4[h.x4off + v]); X[k].w = __uint_as_float(uint32_t(__ldg(&p.pos16[h.x4off + v]))); }
    }
  };

  // the CTA's segment headers and this warp's block counts, cached in shared memory (plan data: before the wait)
  SegHdr *segtab = reinterpret_cast<SegHdr *>(smem + off_segtab(stage_bytes, NW, ring));
  ushort2 *wsegtab = reinterpret_cast<ushort2 *>(smem + off_wsegtab(stage_bytes, NW, ring));
  {
    const int nsc = min(cs.y - cs.x, kSegTab);
    const int4 *src = reinterpret_cast<const int4 *>(p.segs + cs.x);
    for (int i = tid; i < nsc * 2; i += NT) reinterpret_cast<int4 *>(segtab)[i] = __ldg(src + i);
    for (int i = tid; i < nsc * NW; i += NT) wsegtab[i] = __ldg(&p.wseg[size_t(cs.x) * NW + i]);
  }
  auto seg_at = [&](int s) -> SegHdr { return (s - cs.x < kSegTab) ? segtab[s - cs.x] : p.segs[s]; };
  auto wseg_at = [&](int s) -> ushort2 { return (s - cs.x < kSegTab) ? wsegtab[(s - cs.x) * NW + warp] : __ldg(&p.wseg[size_t(s) * NW + warp]); };
  SegHdr hcur{};
  float px[SV][3];
  float4 pX[SV];                    // rest position; .w carries the staging position (bit pattern)
  bool pre = false;                 // (px, pX) hold a prefetched component
  SegHdr h1{};                      // second segment's header (plan data: fetched before the wait as well)
  if (cs.x < cs.y) {
    hcur = p.segs[cs.x];
    if (!GLOBAL && cs.x + 1 < cs.y) h1 = p.segs[cs.x + 1];
    if (!GLOBAL && !hcur.whole) load_rest(hcur, pX);   // first component: plan data, loaded before the wait
  }
  TSB_STAMP(2);
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  TSB_STAMP(3);

  const float gh = p.gradH * (p.gradH_dev ? __ldcg(p.gradH_dev) : 1.f);
  const float s1 = gh * p.c1, s2 = gh * p.c2, s3 = gh * p.c3;
  const bool amips_on = AMIPS && p.c3 != 0.f && p.Bt != nullptr;
  const bool order2 = p.order == 2;
  float *__restrict__ grad = p.grad;
  if (grad) {   // vertices no tet references: zero gradient
    for (int i = blockIdx.x * NT + tid; i < p.n_orphans; i += gridDim.x * NT) {
      const int v = __ldg(&p.orphans[i]);
      grad[3 * size_t(v)] = 0.f; grad[3 * size_t(v) + 1] = 0.f; grad[3 * size_t(v) + 2] = 0.f;
      if constexpr (DIAG && !DET) {   // both planes in one launch
        float *g2 = grad + 3 * size_t(p.n);
        g2[3 * size_t(v)] = 0.f; g2[3 * size_t(v) + 1] = 0.f; g2[3 * size_t(v) + 2] = 0.f;
      }
    }
  }

  double des = 0.0, deb = 0.0, dea = 0.0;     // per-lane energy partials (smoothness, barrier, AMIPS)
  if (SPH && lane == 0) { red[3 * warp] = 0.0; red[3 * warp + 1] = 0.0; red[3 * warp + 2] = 0.0; }
  // LINE: des carries d^T M d and deb u^T M d; lane l keeps the fp64 running sum of tet value line_idx(l) (the warp
  // reduce-scatter below) in dln, and its smallest first root in rmin
  constexpr int kLN = AMIPS ? 2 * kLineMaxAlpha : kLineMaxAlpha;   // tet values: barrier changes, then AMIPS changes
  double dln = 0.0;
  float rmin = INFINITY, amax = 0.f;
  const int nal = LINE ? p.n_alpha : 0;
  if constexpr (LINE)
    for (int k = 0; k < nal; ++k) amax = fmaxf(amax, __ldg(p.alpha + k));

  // staged u = rel_u(x_i, X_i, c) with c = fp32(x_r - X_r) of the component's local vertex r = 0 (tsb_plan.cpp,
  // staging_tables): the component's rigid displacement never enters a rounded difference.  HVP: c = v_r, and the
  // u slots hold v_i - v_r
  auto load_ref = [&](const SegHdr &h, float (&r)[3]) {
    const size_t gr = gid_of(h, 0);
    if constexpr (VS) {
      r[0] = __ldcg(p.v + 3 * gr); r[1] = __ldcg(p.v + 3 * gr + 1); r[2] = __ldcg(p.v + 3 * gr + 2);
    } else {
      const float4 Xr = __ldg(&p.X4[h.x4off]);
      r[0] = __ldcg(p.x + 3 * gr) - Xr.x; r[1] = __ldcg(p.x + 3 * gr + 1) - Xr.y; r[2] = __ldcg(p.x + 3 * gr + 2) - Xr.z;
    }
  };
  // x of a double-buffered component -> registers; HVP: v as well, into X's xyz (its .w, the staging position, stays)
  auto load_x = [&](const SegHdr &h, float (&x)[SV][3], float4 (&X)[SV]) {
#pragma unroll
    for (int k = 0; k < SV; ++k) {
      const int v = tid + k * NT;
      if (v < h.nv) {
        const size_t gi = gid_of(h, v);
        x[k][0] = __ldcg(p.x + 3 * gi); x[k][1] = __ldcg(p.x + 3 * gi + 1); x[k][2] = __ldcg(p.x + 3 * gi + 2);
        if constexpr (VS) { X[k].x = __ldcg(p.v + 3 * gi); X[k].y = __ldcg(p.v + 3 * gi + 1); X[k].z = __ldcg(p.v + 3 * gi + 2); }
      }
    }
  };
  // registers (x, X from load_x / load_rest) -> the component's half-buffer, relative to the reference displacement ref
  auto store_staged_ref = [&](const SegHdr &h, int li, const float (&x)[SV][3], const float4 (&X)[SV], const float (&ref)[3]) {
    float4 *ub = stage + ubase_of(h, li), *xb = stage + xbase_of(h, li);
#pragma unroll
    for (int k = 0; k < SV; ++k) {
      const int v = tid + k * NT;
      if (v < h.nv) {
        const uint32_t pos = VS ? uint32_t(__ldg(&p.pos16[h.x4off + v])) : __float_as_uint(X[k].w);
        if constexpr (VS) ub[pos] = make_float4(X[k].x - ref[0], X[k].y - ref[1], X[k].z - ref[2], 0.f);
        else ub[pos] = make_float4(rel_u(x[k][0], X[k].x, ref[0]), rel_u(x[k][1], X[k].y, ref[1]), rel_u(x[k][2], X[k].z, ref[2]), 0.f);
        xb[pos] = make_float4(x[k][0], x[k][1], x[k][2], 0.f);
      }
    }
  };
  auto store_staged = [&](const SegHdr &h, int li) {
    float pr[3];                            // loaded here, not with px: kept out of the segment loop's live registers
    load_ref(h, pr);
    store_staged_ref(h, li, px, pX, pr);
  };
  auto stage_direct = [&](const SegHdr &h, int li) {   // any size, no register prefetch
    float4 *ub = stage + ubase_of(h, li), *xb = stage + xbase_of(h, li);
    float r[3];
    load_ref(h, r);
    for (int v = tid; v < h.nv; v += NT) {
      const float4 X = __ldg(&p.X4[h.x4off + v]);
      const size_t gi = gid_of(h, v);
      const float x0 = __ldcg(p.x + 3 * gi), x1 = __ldcg(p.x + 3 * gi + 1), x2 = __ldcg(p.x + 3 * gi + 2);
      const uint32_t pos = __ldg(&p.pos16[h.x4off + v]);
      if constexpr (VS) ub[pos] = make_float4(__ldcg(p.v + 3 * gi) - r[0], __ldcg(p.v + 3 * gi + 1) - r[1], __ldcg(p.v + 3 * gi + 2) - r[2], 0.f);
      else ub[pos] = make_float4(rel_u(x0, X.x, r[0]), rel_u(x1, X.y, r[1]), rel_u(x2, X.z, r[2]), 0.f);
      xb[pos] = make_float4(x0, x1, x2, 0.f);
    }
  };

  // The first TWO components are staged before the first barrier (they use different half-buffers), so no
  // CTA-wide barrier separates segments 0 and 1: a warp flows from its work in the first into the second
  // (at <= 64 spheres per GPU no CTA has more than two segments).
  bool eager2 = false;
  if (!GLOBAL) {
    if (cs.x < cs.y) {
      if (cs.x + 1 < cs.y && !hcur.whole) eager2 = !h1.whole;
      if (hcur.whole) {
        stage_direct(hcur, 0);
        ws.request_rest();
      } else if (!eager2) {
        float pr[3];
        load_x(hcur, px, pX); load_ref(hcur, pr);
        ws.request_rest();
        store_staged_ref(hcur, 0, px, pX, pr);
      } else {
        // both components' loads in flight together (second register set), then both stores
        float qx[SV][3], qr[3], pr[3];
        float4 qX[SV];
        load_rest(h1, qX);
        load_x(hcur, px, pX);
        load_ref(h1, qr);
        load_x(h1, qx, qX);
        load_ref(hcur, pr);
        ws.request_rest();
        store_staged_ref(hcur, 0, px, pX, pr);
        store_staged_ref(h1, 1, qx, qX, qr);
      }
    } else {
      ws.request_rest();
    }
    __syncthreads();
    TSB_STAMP(4);
  } else {
    ws.request_rest();
    __syncthreads();      // segment tables visible
  }
  // SPH reads eager2 back from the segment table: it is not kept live through the segment loop (register budget)
  auto eager2_of = [&]() -> bool {
    if constexpr (SPH) return cs.y - cs.x >= 2 && !segtab[0].whole && !segtab[1].whole;
    else return eager2;
  };
  ws.begin();
  TSB_STAMP(12);

  for (int s = cs.x; s < cs.y; ++s) {
    const int li = s - cs.x;
    // ---- prefetch the next component's x / X into registers (lands during this segment's math)
    SegHdr hn{};
    const ushort2 wseg = wseg_at(s);
    pre = false;
    if (s + 1 < cs.y) {
      hn = seg_at(s + 1);
      if (!GLOBAL) {
        const bool e2 = eager2_of();
        pre = !hcur.whole && !hn.whole && !(li == 0 && e2);
        if (pre) {
          load_rest(hn, pX);
          load_x(hn, px, pX);
        }
      }
    }

    // gather of a staged float4.  STAGED: j is a byte offset from the start of shared memory (the plan
    // bakes the segment's half-buffer into it); GLOBAL: j is a vertex id.
    auto gatherU = [&](uint32_t j) -> float4 { return GLOBAL ? __ldg(p.u4g + j) : *reinterpret_cast<const float4 *>(smem + j); };
    auto gatherX = [&](uint32_t j) -> float4 { return GLOBAL ? __ldg(p.x4g + j) : *reinterpret_cast<const float4 *>(smem + j); };
    const int xb16 = GLOBAL ? 0 : xbase_of(hcur, li) * 16;
    auto gid_x = [&](uint32_t j) -> size_t {
      if (GLOBAL) return size_t(j);
      return size_t(__ldg(&p.pos_gid[hcur.p4off + ((j - uint32_t(xb16)) >> 4)]));
    };
    // HVP: staged v - v_ref of the vertex whose x is gathered at j; STAGED: its u slot lies a fixed distance below,
    // formed here (kept live through the row pass, it would cost a register)
    auto gatherV = [&](uint32_t j) -> float4 {
      const uint32_t dv16 = GLOBAL ? 0u : uint32_t(hcur.whole ? hcur.npos : p.vh) * 16u;   // xbase_of - ubase_of
      return gatherU(j - dv16);
    };
    // reference displacement of the component: sum_i g_i = 0, so 1/2 sum_i (u_i - uref).g_i is the same
    // energy with the rigid translation taken out of the cancellation
    const float4 uref = GLOBAL ? __ldg(p.u4g + hcur.x4off) : stage[ubase_of(hcur, li)];
    if (s == cs.x) TSB_STAMP(13);
    // LINE: u^T M d = sum_i (u_i - c).(M d)_i for any c shared by the component (M has zero row and column sums), here
    // c = fp32(x_r - X_r) of the component's reference vertex r, with u_i - c formed by rel_u as the energy stages it.
    // The row's x_i is staged (x slot), its rest position X_i is read by vertex id
    float lc[3] = {0.f, 0.f, 0.f};
    if constexpr (LINE) {
      const size_t gr = GLOBAL ? size_t(hcur.x4off) : gid_of(hcur, 0);
      const float4 Xr = __ldg(&p.X4[hcur.x4off]);
      lc[0] = __ldcg(p.x + 3 * gr) - Xr.x; lc[1] = __ldcg(p.x + 3 * gr + 1) - Xr.y; lc[2] = __ldcg(p.x + 3 * gr + 2) - Xr.z;
    }
    auto rest_of = [&](uint32_t rid) -> float4 {
      if (GLOBAL) return __ldg(&p.X4[rid]);
      if (hcur.vbase >= 0) return __ldg(&p.X4[hcur.x4off + int(rid) - hcur.vbase]);
      // a component's vertices are staged in ascending id order: binary search of its vlist range
      int lo = 0, hi = hcur.nv - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (uint32_t(__ldg(&p.vlist[hcur.x4off + mid])) < rid) lo = mid + 1; else hi = mid;
      }
      return __ldg(&p.X4[hcur.x4off + lo]);
    };

    // ---- operator rows: L lanes per vertex row (header in slot 0 of the first quad) ------------------
    for (int rb = 0; rb < int(wseg.x); ++rb) {
      const uint32_t hdr = *reinterpret_cast<const uint32_t *>(ws.cell + WOFF + lane * 16);
      const uint32_t rid = hdr & 0xFFFFFFu, len4 = (hdr >> 24) & 63u, llog = hdr >> 30;   // global row id | quads | log2(lanes per row)
      const bool active = rid != 0xFFFFFFu;
      const uint32_t rowj = GLOBAL ? *reinterpret_cast<const uint32_t *>(ws.cell + lane * 16)
                                   : uint32_t(*reinterpret_cast<const uint16_t *>(ws.cell + lane * 8));
      const float4 ui = DIAG ? make_float4(0.f, 0.f, 0.f, 0.f) : gatherU(rowj);
      f32x2 AX{0.f, 0.f}, AY{0.f, 0.f}, AZ{0.f, 0.f};     // (even-entry, odd-entry) partial sums
      uint32_t left = len4;
      while (left) {
        const uint32_t n = min(left, ws.avail());
        const unsigned char *cp = ws.cell + lane * 4 * F::IB;
#pragma unroll 2
        for (uint32_t q = 0; q < n; ++q, cp += CELL) {
          uint32_t j[4];
          if (GLOBAL) {
            const uint4 qi = *reinterpret_cast<const uint4 *>(cp);
            j[0] = qi.x; j[1] = qi.y; j[2] = qi.z; j[3] = qi.w;
          } else {
            const uint2 qi = *reinterpret_cast<const uint2 *>(cp);
            j[0] = qi.x & 0xFFFFu; j[1] = qi.x >> 16; j[2] = qi.y & 0xFFFFu; j[3] = qi.y >> 16;
          }
          const float4 qw = *reinterpret_cast<const float4 *>(cp + WOFF + lane * (16 - 4 * F::IB));
          if constexpr (DIAG) {
            // the row's off-diagonal weights M_ij; an entry whose column is the row itself is the lane's header slot
            // (its weight is the header's bit pattern) and adds nothing, as it adds nothing to M u
            AX.lo += j[0] != rowj ? qw.x : 0.f; AX.hi += j[1] != rowj ? qw.y : 0.f;
            AX.lo += j[2] != rowj ? qw.z : 0.f; AX.hi += j[3] != rowj ? qw.w : 0.f;
            continue;
          }
          const float4 u0 = gatherU(j[0]), u1 = gatherU(j[1]), u2 = gatherU(j[2]), u3 = gatherU(j[3]);
          const f32x2 W01 = pk2(qw.x, qw.y), W23 = pk2(qw.z, qw.w);
          fma2_acc(AX, W01, pk2(u0.x - ui.x, u1.x - ui.x));
          fma2_acc(AY, W01, pk2(u0.y - ui.y, u1.y - ui.y));
          fma2_acc(AZ, W01, pk2(u0.z - ui.z, u1.z - ui.z));
          fma2_acc(AX, W23, pk2(u2.x - ui.x, u3.x - ui.x));
          fma2_acc(AY, W23, pk2(u2.y - ui.y, u3.y - ui.y));
          fma2_acc(AZ, W23, pk2(u2.z - ui.z, u3.z - ui.z));
        }
        ws.advance(n);
        left -= n;
      }
#ifdef TSB_TRACE
      if (s == cs.x && rb == 0) { TSB_STAMP(14); if (tid == 0 && p.trace) p.trace[blockIdx.x * kTraceSlots + 15] = len4 | (uint32_t(wseg.x) << 16) | (uint32_t(wseg.y) << 24); }
#endif
      float ax = sum2(AX), ay = sum2(AY), az = sum2(AZ);
      for (uint32_t o = 1; o < (1u << llog); o <<= 1) {   // the L lanes of a row are adjacent
        ax += __shfl_xor_sync(0xffffffffu, ax, o);
        if constexpr (!DIAG) {
          ay += __shfl_xor_sync(0xffffffffu, ay, o);
          az += __shfl_xor_sync(0xffffffffu, az, o);
        }
      }
      if (DIAG && active && (lane & ((1u << llog) - 1u)) == 0) {
        // plane 0: s1 M_ii (1, 1, 1) with M_ii = -sum_{j != i} M_ij (M has zero row sums); plane 1: 0.  DET: the plane
        // of this launch
        const size_t gi = rid;
        const float d = (DET && p.diag_plane) ? 0.f : -(s1 * ax);
        grad[3 * gi] = d; grad[3 * gi + 1] = d; grad[3 * gi + 2] = d;
        if constexpr (!DET) {
          float *g2 = grad + 3 * size_t(p.n);
          g2[3 * gi] = 0.f; g2[3 * gi + 1] = 0.f; g2[3 * gi + 2] = 0.f;
        }
      } else if (!DIAG && active && (lane & ((1u << llog) - 1u)) == 0) {
        des += double(fmaf(ui.x - uref.x, ax, fmaf(ui.y - uref.y, ay, (ui.z - uref.z) * az)));
        if constexpr (LINE) {
          const uint32_t dv16 = GLOBAL ? 0u : uint32_t(hcur.whole ? hcur.npos : p.vh) * 16u;   // as gatherV
          const float4 xi = gatherX(rowj + dv16), Xi = rest_of(rid);
          deb += double(fmaf(rel_u(xi.x, Xi.x, lc[0]), ax, fmaf(rel_u(xi.y, Xi.y, lc[1]), ay, rel_u(xi.z, Xi.z, lc[2]) * az)));
        }
        if (grad) {
          const size_t gi = rid;
          grad[3 * gi] = s1 * ax; grad[3 * gi + 1] = s1 * ay; grad[3 * gi + 2] = s1 * az;
        }
      }
    }
    if (s == cs.x) TSB_STAMP(5);
    if (!DET && grad) {   // all warps' rows of this segment are stored -> ONE release of the component's counter, sent by
                  // the last warp (which owns no tets, so it never waits on its own signal)
      const int bar_id = 1 + (li & 1);      // segments 0 and 1 may be in flight together: two barrier ids
      if (warp == NW - 1) {
        asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "n"(NT) : "memory");
        if (lane == 0) { __threadfence(); atomicAdd(p.done + hcur.comp, 1u); }
      } else {
        asm volatile("bar.arrive %0, %1;" ::"r"(bar_id), "n"(NT) : "memory");
      }
    }

    // ---- barrier: TPL tets per lane ---------------------------------------------------------------------
    bool waited = false;
    auto wait_rows = [&] {   // every row of this component must be stored before we add to it
      if (!waited) {
        const unsigned int need = unsigned(hcur.expected);
        while (ld_acquire(p.done + hcur.comp) < need) __nanosleep(40);
        waited = true;
      }
    };
    const int tcell0 = (amips_on || (DET && grad)) ? __ldg(&p.wtc0[size_t(s) * NW + warp]) : 0;
    // DET: corner vectors c0..c3 of the tet in slot lane * TPL + t of tet cell tcell0 + tc
    auto det_store = [&](int tc, int t, float c0x, float c0y, float c0z, float c1x, float c1y, float c1z, float c2x, float c2y,
                         float c2z, float c3x, float c3y, float c3z) {
      float4 *d = p.det_scratch + 3 * (size_t(tcell0 + tc) * (32 * F::TPL) + lane * F::TPL + t);
      d[0] = make_float4(c0x, c0y, c0z, c1x);
      d[1] = make_float4(c1y, c1z, c2x, c2y);
      d[2] = make_float4(c2z, c3x, c3y, c3z);
    };
    int mnK = 0x7F800000;   // SPH: the warp's smallest J of a real tet in the segment (as an int key), its J < 0 count
    int nneg = 0;
    for (int tc = 0; tc < int(wseg.y); ++tc) {
      uint32_t dmask = 0;   // DET: bit t = this lane's tet t contributed
      float lv[kLN];        // LINE: this lane's tets' changes per alpha (barrier, then AMIPS), summed over the cell
#pragma unroll
      for (int i = 0; i < kLN; ++i) lv[i] = 0.f;
      uint32_t tj[F::TPL][4];
      float tdet[F::TPL];
      if (GLOBAL) {
        const uint4 a = *reinterpret_cast<const uint4 *>(ws.cell + lane * 16);
        tj[0][0] = a.x; tj[0][1] = a.y; tj[0][2] = a.z; tj[0][3] = a.w;
        tdet[0] = *reinterpret_cast<const float *>(ws.cell + 512 + lane * 4);
      } else {
        const uint4 a = *reinterpret_cast<const uint4 *>(ws.cell + lane * 16);
        const float2 d = *reinterpret_cast<const float2 *>(ws.cell + 512 + lane * 8);
        tj[0][0] = a.x & 0xFFFFu; tj[0][1] = a.x >> 16; tj[0][2] = a.y & 0xFFFFu; tj[0][3] = a.y >> 16;
        tj[F::TPL - 1][0] = a.z & 0xFFFFu; tj[F::TPL - 1][1] = a.z >> 16; tj[F::TPL - 1][2] = a.w & 0xFFFFu; tj[F::TPL - 1][3] = a.w >> 16;
        tdet[0] = d.x; tdet[F::TPL - 1] = d.y;
      }
      // HVP or DIAG with AMIPS: a lane's later tets gather their corners when they are reached, so that those registers
      // are free for the AMIPS product or blocks (the staging area and x4g stay valid for the whole segment)
      constexpr bool kLateX = (HVP || DIAG) && AMIPS;
      float4 xv[F::TPL][4];
#pragma unroll
      for (int t = 0; t < int(F::TPL); ++t)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (!kLateX || t == 0) xv[t][k] = gatherX(tj[t][k]);
      ws.advance(1);
#pragma unroll
      for (int t = 0; t < int(F::TPL); ++t) {
        if (kLateX && t > 0)
#pragma unroll
          for (int k = 0; k < 4; ++k) xv[t][k] = gatherX(tj[t][k]);
        const float4 x0 = xv[t][0], x1 = xv[t][1], x2 = xv[t][2], x3 = xv[t][3];
        const float idet = tdet[t];
        const float e1x = x1.x - x0.x, e1y = x1.y - x0.y, e1z = x1.z - x0.z;
        const float e2x = x2.x - x0.x, e2y = x2.y - x0.y, e2z = x2.z - x0.z;
        const float e3x = x3.x - x0.x, e3y = x3.y - x0.y, e3z = x3.z - x0.z;
        const float c1x = e2y * e3z - e2z * e3y, c1y = e2z * e3x - e2x * e3z, c1z = e2x * e3y - e2y * e3x;   // e2 x e3
        const float J = (e1x * c1x + e1y * c1y + e1z * c1z) * idet;
        if constexpr (SPH) {
          // warp-uniform accumulators (no per-lane register).  J as an int key whose signed order is J's order;
          // padding tets (1/det(Dm) = 0, J = 0) are not part of the sphere and enter as +inf
          const int kJ = idet == 0.f ? 0x7F800000 : (__float_as_int(J) < 0 ? __float_as_int(J) ^ 0x7FFFFFFF : __float_as_int(J));
          mnK = min(mnK, __reduce_min_sync(0xffffffffu, kJ));
          nneg += __popc(__ballot_sync(0xffffffffu, J < 0.f));
        }
        if constexpr (DIAG) {
          // Diagonal block of corner k: D_k = al |b_k|^2 I + be (g f^T + f g^T) + ga g g^T, g = dJ/dx_k = idet c_k (the
          // gradient's corner vector; g_0 = -(g_1 + g_2 + g_3)).  Barrier (J < 0, m = -J): J is multilinear in the
          // corners, so d2J/dx_k^2 = 0 and al = be = 0, ga = s2 p (p-1) m^(p-2).  AMIPS (J > 0): moving corner k gives
          // dF = delta b_k^T (b_k: row k of B = Dm^-1, b_0 = -sum), f = F b_k, a = 2 / (3 J^(2/3)): al = s3 a,
          // be = -2 al / (3 J), ga = 5 al I1 / (9 J^2)   (DESIGN.md section 5, "Hessian diagonal")
          if (J < 0.f || (AMIPS && amips_on && J > 0.f)) {
            float al = 0.f, be = 0.f, ga;
            float Fm[3][3] = {}, bb[3][3] = {};
            if (J < 0.f) {
              const float m = -J;
              ga = s2 * (order2 ? 2.f : 12.f * m * m);
            } else {
              const int slot = lane * int(F::TPL) + t;
              const float4 *bp = p.Bt + (size_t(tcell0 + tc) * 3) * (32 * F::TPL) + slot;
              const float4 b0 = __ldg(bp), b1 = __ldg(bp + 32 * F::TPL), b2 = __ldg(bp + 64 * F::TPL);
              bb[0][0] = b0.x; bb[0][1] = b0.y; bb[0][2] = b0.z;
              bb[1][0] = b1.x; bb[1][1] = b1.y; bb[1][2] = b1.z;
              bb[2][0] = b2.x; bb[2][1] = b2.y; bb[2][2] = b2.z;
              const float ex[3] = {e1x, e2x, e3x}, ey[3] = {e1y, e2y, e3y}, ez[3] = {e1z, e2z, e3z};
              float tr = 0.f;
#pragma unroll
              for (int c = 0; c < 3; ++c) {
                Fm[0][c] = ex[0] * bb[0][c] + ex[1] * bb[1][c] + ex[2] * bb[2][c];
                Fm[1][c] = ey[0] * bb[0][c] + ey[1] * bb[1][c] + ey[2] * bb[2][c];
                Fm[2][c] = ez[0] * bb[0][c] + ez[1] * bb[1][c] + ez[2] * bb[2][c];
                tr = fmaf(Fm[0][c], Fm[0][c], fmaf(Fm[1][c], Fm[1][c], fmaf(Fm[2][c], Fm[2][c], tr)));
              }
              const float cb = cbrtf(J), iJ = 1.f / J;
              al = s3 * (2.f / (3.f * (cb * cb)));
              be = -(2.f / 3.f) * al * iJ;
              ga = (5.f / 9.f) * al * tr * (iJ * iJ);
            }
            // the six entries of D_k: (xx, yy, zz) for plane 0, (yz, xz, xy) for plane 1
            auto block = [&](const float (&g)[3], const float (&f)[3], float b2, float (&o)[6]) {
#pragma unroll
              for (int r = 0; r < 3; ++r) o[r] = fmaf(al, b2, fmaf(2.f * be * g[r], f[r], ga * g[r] * g[r]));
              o[3] = fmaf(be, fmaf(g[1], f[2], f[1] * g[2]), ga * g[1] * g[2]);
              o[4] = fmaf(be, fmaf(g[0], f[2], f[0] * g[2]), ga * g[0] * g[2]);
              o[5] = fmaf(be, fmaf(g[0], f[1], f[0] * g[1]), ga * g[0] * g[1]);
            };
            const bool pl = DET && p.diag_plane;
            float keep[4][3];   // DET: this launch's plane of every corner
            auto emit = [&](int k, const float (&o)[6]) {
              if constexpr (DET) {
#pragma unroll
                for (int r = 0; r < 3; ++r) keep[k][r] = pl ? o[3 + r] : o[r];
              } else {
                const size_t vk = 3 * gid_x(tj[t][k]);
                float *g2 = grad + 3 * size_t(p.n);
#pragma unroll
                for (int r = 0; r < 3; ++r) { atomicAdd(grad + vk + r, o[r]); atomicAdd(g2 + vk + r, o[3 + r]); }
              }
            };
            if constexpr (DET) dmask |= 1u << t;
            else wait_rows();
            // corner k = 0..3: the edge pair (a, b) of c_k = a x b, with c_0 = -(c1 + c2 + c3) = (e3 - e1) x (e2 - e1)
            // (c1 = e2 x e3, c2 = e3 x e1, c3 = e1 x e2), and b_k (b_0 = -(b_1 + b_2 + b_3))
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float ax = k == 0 ? e3x - e1x : (k == 1 ? e2x : (k == 2 ? e3x : e1x));
              const float ay = k == 0 ? e3y - e1y : (k == 1 ? e2y : (k == 2 ? e3y : e1y));
              const float az = k == 0 ? e3z - e1z : (k == 1 ? e2z : (k == 2 ? e3z : e1z));
              const float bx = k == 0 ? e2x - e1x : (k == 1 ? e3x : (k == 2 ? e1x : e2x));
              const float by = k == 0 ? e2y - e1y : (k == 1 ? e3y : (k == 2 ? e1y : e2y));
              const float bz = k == 0 ? e2z - e1z : (k == 1 ? e3z : (k == 2 ? e1z : e2z));
              const float g[3] = {idet * (ay * bz - az * by), idet * (az * bx - ax * bz), idet * (ax * by - ay * bx)};
              float bk[3];
#pragma unroll
              for (int c = 0; c < 3; ++c) bk[c] = k == 0 ? -(bb[0][c] + bb[1][c] + bb[2][c]) : bb[k - 1][c];
              float f[3];
#pragma unroll
              for (int r = 0; r < 3; ++r) f[r] = Fm[r][0] * bk[0] + Fm[r][1] * bk[1] + Fm[r][2] * bk[2];
              float o[6];
              block(g, f, bk[0] * bk[0] + bk[1] * bk[1] + bk[2] * bk[2], o);
              emit(k, o);
            }
            if constexpr (DET)
              det_store(tc, t, keep[0][0], keep[0][1], keep[0][2], keep[1][0], keep[1][1], keep[1][2], keep[2][0], keep[2][1],
                        keep[2][2], keep[3][0], keep[3][1], keep[3][2]);
          }
        } else if constexpr (LINE) {
          // det F(x + alpha d) = J + alpha (J1 + alpha (J2 + alpha J3)): with the edges e_k of x and f_k of d,
          // J1 = idet f.cof E = idet sum_k f_k.c_k (c1 = e2 x e3, c2 = e3 x e1, c3 = e1 x e2), J2 = idet e.cof(f)
          // = idet sum_k e_k.g_k (g1 = f2 x f3, ...), J3 = idet f1.g1
          const float4 w0 = gatherV(tj[t][0]), w1 = gatherV(tj[t][1]), w2 = gatherV(tj[t][2]), w3 = gatherV(tj[t][3]);
          const float f1x = w1.x - w0.x, f1y = w1.y - w0.y, f1z = w1.z - w0.z;
          const float f2x = w2.x - w0.x, f2y = w2.y - w0.y, f2z = w2.z - w0.z;
          const float f3x = w3.x - w0.x, f3y = w3.y - w0.y, f3z = w3.z - w0.z;
          const float g1x = f2y * f3z - f2z * f3y, g1y = f2z * f3x - f2x * f3z, g1z = f2x * f3y - f2y * f3x;
          const float J1 = (f1x * c1x + f1y * c1y + f1z * c1z + f2x * (e3y * e1z - e3z * e1y) + f2y * (e3z * e1x - e3x * e1z) +
                            f2z * (e3x * e1y - e3y * e1x) + f3x * (e1y * e2z - e1z * e2y) + f3y * (e1z * e2x - e1x * e2z) +
                            f3z * (e1x * e2y - e1y * e2x)) * idet;
          const float J2 = (e1x * g1x + e1y * g1y + e1z * g1z + e2x * (f3y * f1z - f3z * f1y) + e2y * (f3z * f1x - f3x * f1z) +
                            e2z * (f3x * f1y - f3y * f1x) + e3x * (f1y * f2z - f1z * f2y) + e3y * (f1z * f2x - f1x * f2z) +
                            e3z * (f1x * f2y - f1y * f2x)) * idet;
          const float J3 = (f1x * g1x + f1y * g1y + f1z * g1z) * idet;
          auto dJ_at = [&](float al) { return al * fmaf(al, fmaf(al, J3, J2), J1); };   // J(al) - J, so J(0) = J
          // AMIPS: I1(alpha) = |F + alpha dF|^2 = tr + alpha (2 fdf + alpha dd), F = E B, dF = f B
          float tr = 0.f, fdf = 0.f, dd = 0.f, r0 = 0.f;
          if (AMIPS && amips_on) {
            const int slot = lane * int(F::TPL) + t;
            const float4 *bp = p.Bt + (size_t(tcell0 + tc) * 3) * (32 * F::TPL) + slot;
            const float4 b0 = __ldg(bp), b1 = __ldg(bp + 32 * F::TPL), b2 = __ldg(bp + 64 * F::TPL);
            const float bb[3][3] = {{b0.x, b0.y, b0.z}, {b1.x, b1.y, b1.z}, {b2.x, b2.y, b2.z}};
            const float ex[3] = {e1x, e2x, e3x}, ey[3] = {e1y, e2y, e3y}, ez[3] = {e1z, e2z, e3z};
            const float fx[3] = {f1x, f2x, f3x}, fy[3] = {f1y, f2y, f3y}, fz[3] = {f1z, f2z, f3z};
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const float F0 = ex[0] * bb[0][c] + ex[1] * bb[1][c] + ex[2] * bb[2][c];
              const float F1 = ey[0] * bb[0][c] + ey[1] * bb[1][c] + ey[2] * bb[2][c];
              const float F2 = ez[0] * bb[0][c] + ez[1] * bb[1][c] + ez[2] * bb[2][c];
              const float D0 = fx[0] * bb[0][c] + fx[1] * bb[1][c] + fx[2] * bb[2][c];
              const float D1 = fy[0] * bb[0][c] + fy[1] * bb[1][c] + fy[2] * bb[2][c];
              const float D2 = fz[0] * bb[0][c] + fz[1] * bb[1][c] + fz[2] * bb[2][c];
              tr = fmaf(F0, F0, fmaf(F1, F1, fmaf(F2, F2, tr)));
              fdf = fmaf(F0, D0, fmaf(F1, D1, fmaf(F2, D2, fdf)));
              dd = fmaf(D0, D0, fmaf(D1, D1, fmaf(D2, D2, dd)));
            }
            if (J > 0.f) r0 = cbrtf(J);
          }
#pragma unroll
          for (int k = 0; k < kLineMaxAlpha; ++k) {
            if (k < nal) {
              const float al = __ldg(p.alpha + k);
              const float dJ = dJ_at(al), Ja = J + dJ;
              // barrier: with both ends inverted m^p - m0^p = (m - m0)(m + m0)[(m^2 + m0^2)], m - m0 = -dJ
              const float m0 = fmaxf(-J, 0.f), m = fmaxf(-Ja, 0.f);
              float db;
              if (Ja < 0.f && J < 0.f) {
                const float q = -dJ * (m + m0);
                db = order2 ? q : q * fmaf(m, m, m0 * m0);
              } else {
                const float mm = m * m, mm0 = m0 * m0;   // at most one of them is nonzero
                db = order2 ? mm - mm0 : mm * mm - mm0 * mm0;
              }
              lv[k] += db;
              if (AMIPS && amips_on) {
                // psi = I1 / (3 J^(2/3)) - 1 where J > 0.  Both ends active: with r = J(alpha)^(1/3), r0 = J^(1/3),
                // psi(alpha) - psi(0) = dI1 / (3 r^2) - I1(0) dJ (r0 + r) / (3 r^2 r0^2 (r^2 + r r0 + r0^2)),
                // free of the cancellation of two psi values near 1
                float da = 0.f;
                const float dI = al * fmaf(al, dd, 2.f * fdf);
                if (Ja > 0.f) {
                  const float r = cbrtf(Ja), r2 = r * r, q = 1.f / (3.f * r2);
                  if (J > 0.f) {
                    const float r02 = r0 * r0;
                    da = dI * q - tr * dJ * (r0 + r) * q / (r02 * fmaf(r, r + r0, r02));
                  } else {
                    da = (tr + dI) * q - 1.f;
                  }
                } else if (J > 0.f) {
                  da = 1.f - tr / (3.f * (r0 * r0));
                }
                lv[kLineMaxAlpha + k] += da;
              }
            }
          }
          // first root of J(alpha) in (0, amax] for a real tet with J > 0 (padding tets have idet = 0, so J = 0): split
          // [0, amax] at the roots of J' = J1 + 2 J2 a + 3 J3 a^2 into monotone pieces, find the first piece whose end
          // has J <= 0 (or a critical point where J is within rounding of 0: a double root), then bisect it on the
          // float's bit pattern (nonnegative floats order as their bits: 32 halvings reach adjacent floats at any scale)
          float lo = 0.f, hi = -1.f;
          if (J > 0.f && amax > 0.f) {
            float q1 = 0.f, q2 = 0.f;    // critical points in (0, amax), ascending; 0 = none
            if (J3 != 0.f) {
              const float A = 3.f * J3, Bq = 2.f * J2;
              const float D = fmaf(Bq, Bq, -4.f * A * J1);
              if (D > 0.f) {
                const float qq = -0.5f * (Bq + copysignf(sqrtf(D), Bq));
                const float ra = qq / A, rb = qq != 0.f ? J1 / qq : ra;
                q1 = fminf(ra, rb); q2 = fmaxf(ra, rb);
              }
            } else if (J2 != 0.f) {
              q1 = -J1 / (2.f * J2);
            }
            q1 = (q1 > 0.f && q1 < amax) ? q1 : 0.f;
            q2 = (q2 > 0.f && q2 < amax) ? q2 : 0.f;
            const float ends[3] = {q1, q2, amax};
#pragma unroll
            for (int i = 0; i < 3; ++i) {
              const float e = ends[i];
              if (hi < 0.f && e > lo) {
                const float Je = J + dJ_at(e);
                const float tol = i < 2 ? 4.8e-7f * (fabsf(J) + e * (fabsf(J1) + e * (fabsf(J2) + e * fabsf(J3)))) : 0.f;
                if (Je <= tol) { hi = e; if (Je > 0.f) lo = e; }
                else lo = e;
              }
            }
          }
          if (__any_sync(0xffffffffu, hi >= 0.f)) {
            uint32_t a = hi >= 0.f ? __float_as_uint(lo) : 0u, b = hi >= 0.f ? __float_as_uint(hi) : 0u;
#pragma unroll 4
            for (int it = 0; it < 32; ++it) {
              const uint32_t mid = a + ((b - a) >> 1);
              const bool pos = J + dJ_at(__uint_as_float(mid)) > 0.f;
              a = pos ? mid : a;
              b = pos ? b : mid;
            }
            if (hi >= 0.f) rmin = fminf(rmin, __uint_as_float(a));
          }
        } else if (HVP && J < 0.f) {
          // H_t v = phi''(J) dJ g + phi'(J) dg with g_k = dJ/dx_k, dJ = sum_k g_k.f_k and dg_k its derivative along v
          // (f_k = v_k - v_0); phi = (-J)^p.  v^T H_t v = sum_{k=1..3} f_k.(H_t v)_k
          const float m = -J, m2 = m * m;
          const float4 w0 = gatherV(tj[t][0]), w1 = gatherV(tj[t][1]), w2 = gatherV(tj[t][2]), w3 = gatherV(tj[t][3]);
          const float f1x = w1.x - w0.x, f1y = w1.y - w0.y, f1z = w1.z - w0.z;
          const float f2x = w2.x - w0.x, f2y = w2.y - w0.y, f2z = w2.z - w0.z;
          const float f3x = w3.x - w0.x, f3y = w3.y - w0.y, f3z = w3.z - w0.z;
          // (H_t v)_k = a c_k - b dc_k with c1 = e2 x e3, c2 = e3 x e1, c3 = e1 x e2 and their derivatives along v
          // dc1 = f2 x e3 + e2 x f3, dc2 = f3 x e1 + e3 x f1, dc3 = f1 x e2 + e1 x f2.  dJ det(Dm) = f1.c1 + f2.c2 + f3.c3
          // = f1.c1 + e1.dc1, so each k needs only its own c_k, dc_k (fewer live registers)
          const float d1x = (f2y * e3z - f2z * e3y) + (e2y * f3z - e2z * f3y);
          const float d1y = (f2z * e3x - f2x * e3z) + (e2z * f3x - e2x * f3z);
          const float d1z = (f2x * e3y - f2y * e3x) + (e2x * f3y - e2y * f3x);
          const float dJ = (f1x * c1x + f1y * c1y + f1z * c1z + e1x * d1x + e1y * d1y + e1z * d1z) * idet;
          const float a = (order2 ? 2.f : 12.f * m2) * dJ * idet;    // p (p-1) (-J)^(p-2) dJ / det(Dm)
          const float b = (order2 ? 2.f * m : 4.f * m2 * m) * idet;  // p (-J)^(p-1) / det(Dm)
          // corner k of gradH c2 H_t v leaves as soon as it is formed (register budget): DET into the tet slot's 12 floats
          // (the layout det_store writes), otherwise added to hv after the component's rows
          if constexpr (DET) dmask |= 1u << t;
          else wait_rows();
          float *dst = reinterpret_cast<float *>(p.det_scratch + 3 * (size_t(tcell0 + tc) * (32 * F::TPL) + lane * F::TPL + t));
          float g0x = 0.f, g0y = 0.f, g0z = 0.f;
          float q = 0.f;
          auto put = [&](int k, float hx, float hy, float hz, float fx, float fy, float fz) {
            q += fx * hx + fy * hy + fz * hz;
            const float gx = s2 * hx, gy = s2 * hy, gz = s2 * hz;
            g0x -= gx; g0y -= gy; g0z -= gz;
            if constexpr (DET) { dst[3 * k] = gx; dst[3 * k + 1] = gy; dst[3 * k + 2] = gz; }
            else { const size_t vk = 3 * gid_x(tj[t][k]); atomicAdd(grad + vk, gx); atomicAdd(grad + vk + 1, gy); atomicAdd(grad + vk + 2, gz); }
          };
          put(1, a * c1x - b * d1x, a * c1y - b * d1y, a * c1z - b * d1z, f1x, f1y, f1z);
          put(2, a * (e3y * e1z - e3z * e1y) - b * ((f3y * e1z - f3z * e1y) + (e3y * f1z - e3z * f1y)),
              a * (e3z * e1x - e3x * e1z) - b * ((f3z * e1x - f3x * e1z) + (e3z * f1x - e3x * f1z)),
              a * (e3x * e1y - e3y * e1x) - b * ((f3x * e1y - f3y * e1x) + (e3x * f1y - e3y * f1x)), f2x, f2y, f2z);
          put(3, a * (e1y * e2z - e1z * e2y) - b * ((f1y * e2z - f1z * e2y) + (e1y * f2z - e1z * f2y)),
              a * (e1z * e2x - e1x * e2z) - b * ((f1z * e2x - f1x * e2z) + (e1z * f2x - e1x * f2z)),
              a * (e1x * e2y - e1y * e2x) - b * ((f1x * e2y - f1y * e2x) + (e1x * f2y - e1y * f2x)), f3x, f3y, f3z);
          deb += double(q);   // v^T H_t v
          if constexpr (DET) { dst[0] = g0x; dst[1] = g0y; dst[2] = g0z; }
          else { const size_t v0 = 3 * gid_x(tj[t][0]); atomicAdd(grad + v0, g0x); atomicAdd(grad + v0 + 1, g0y); atomicAdd(grad + v0 + 2, g0z); }
        } else if (!HVP && J < 0.f) {
          const float m = -J, m2 = m * m;
          deb += double(order2 ? m2 : m2 * m2);
          if (grad) {
            const float coef = order2 ? 2.f * m : 4.f * m2 * m;       // p (-J)^(p-1)
            const float k = -coef * idet * s2;                         // gradH c2 dphi/dJ / det(Dm)
            const float g1x = k * c1x, g1y = k * c1y, g1z = k * c1z;
            const float g2x = k * (e3y * e1z - e3z * e1y), g2y = k * (e3z * e1x - e3x * e1z), g2z = k * (e3x * e1y - e3y * e1x);
            const float g3x = k * (e1y * e2z - e1z * e2y), g3y = k * (e1z * e2x - e1x * e2z), g3z = k * (e1x * e2y - e1y * e2x);
            if constexpr (DET) {
              det_store(tc, t, -(g1x + g2x + g3x), -(g1y + g2y + g3y), -(g1z + g2z + g3z), g1x, g1y, g1z, g2x, g2y, g2z, g3x, g3y, g3z);
              dmask |= 1u << t;
              continue;
            }
            wait_rows();
            const size_t v0 = 3 * gid_x(tj[t][0]), v1 = 3 * gid_x(tj[t][1]), v2 = 3 * gid_x(tj[t][2]), v3 = 3 * gid_x(tj[t][3]);
            atomicAdd(grad + v0, -(g1x + g2x + g3x)); atomicAdd(grad + v0 + 1, -(g1y + g2y + g3y)); atomicAdd(grad + v0 + 2, -(g1z + g2z + g3z));
            atomicAdd(grad + v1, g1x); atomicAdd(grad + v1 + 1, g1y); atomicAdd(grad + v1 + 2, g1z);
            atomicAdd(grad + v2, g2x); atomicAdd(grad + v2 + 1, g2y); atomicAdd(grad + v2 + 2, g2z);
            atomicAdd(grad + v3, g3x); atomicAdd(grad + v3 + 1, g3y); atomicAdd(grad + v3 + 2, g3z);
          }
        } else if (HVP && AMIPS && amips_on && J > 0.f) {
          // H_a v of AMIPS (tsb_hvp_ex): with dF = dDs B (dDs columns f_k = v_k - v_0), a = 2 / (3 J^(2/3)),
          // beta = tr / (3 J) and C = cof F:  dJ = C:dF,  da = -2/3 a dJ / J,  dbeta = (2 F:dF - tr dJ / J) / (3 J),
          // dC = cof_pair(F, dF) + cof_pair(dF, F),  dP = da (F - beta C) + a (dF - dbeta C - beta dC).  Corner k + 1
          // is dP (row k of B)^T, corner 0 minus their sum; v^T H_a v = sum_t dF:dP (DESIGN.md section 5)
          const int slot = lane * int(F::TPL) + t;
          const float4 *bp = p.Bt + (size_t(tcell0 + tc) * 3) * (32 * F::TPL) + slot;
          const float4 b0 = __ldg(bp), b1 = __ldg(bp + 32 * F::TPL), b2 = __ldg(bp + 64 * F::TPL);
          const float4 w0 = gatherV(tj[t][0]), w1 = gatherV(tj[t][1]), w2 = gatherV(tj[t][2]), w3 = gatherV(tj[t][3]);
          const float ex[3] = {e1x, e2x, e3x}, ey[3] = {e1y, e2y, e3y}, ez[3] = {e1z, e2z, e3z};
          const float fx[3] = {w1.x - w0.x, w2.x - w0.x, w3.x - w0.x}, fy[3] = {w1.y - w0.y, w2.y - w0.y, w3.y - w0.y};
          const float fz[3] = {w1.z - w0.z, w2.z - w0.z, w3.z - w0.z};
          const float bb[3][3] = {{b0.x, b0.y, b0.z}, {b1.x, b1.y, b1.z}, {b2.x, b2.y, b2.z}};
          float Fm[3][3], dF[3][3];
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            Fm[0][c] = ex[0] * bb[0][c] + ex[1] * bb[1][c] + ex[2] * bb[2][c];
            Fm[1][c] = ey[0] * bb[0][c] + ey[1] * bb[1][c] + ey[2] * bb[2][c];
            Fm[2][c] = ez[0] * bb[0][c] + ez[1] * bb[1][c] + ez[2] * bb[2][c];
            dF[0][c] = fx[0] * bb[0][c] + fx[1] * bb[1][c] + fx[2] * bb[2][c];
            dF[1][c] = fy[0] * bb[0][c] + fy[1] * bb[1][c] + fy[2] * bb[2][c];
            dF[2][c] = fz[0] * bb[0][c] + fz[1] * bb[1][c] + fz[2] * bb[2][c];
          }
          // cofactor entries are recomputed where used (register budget): cof_pair(A, B)[r][c] =
          // A[r+1][c+1] B[r+2][c+2] - A[r+1][c+2] B[r+2][c+1], indices mod 3
          auto cofp = [](const float (&A)[3][3], const float (&Bm)[3][3], int r, int c) -> float {
            const int r1 = (r + 1) % 3, r2 = (r + 2) % 3, c1 = (c + 1) % 3, c2 = (c + 2) % 3;
            return A[r1][c1] * Bm[r2][c2] - A[r1][c2] * Bm[r2][c1];
          };
          float tr = 0.f, fdf = 0.f, dJ = 0.f;
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              tr = fmaf(Fm[r][c], Fm[r][c], tr);
              fdf = fmaf(Fm[r][c], dF[r][c], fdf);
              dJ = fmaf(cofp(Fm, Fm, r, c), dF[r][c], dJ);
            }
          const float cb = cbrtf(J), j23 = cb * cb, iJ = 1.f / J;
          const float a = 2.f / (3.f * j23), bq = tr * (1.f / 3.f) * iJ;
          const float da = -(2.f / 3.f) * a * dJ * iJ;
          const float dbq = (2.f * fdf - tr * dJ * iJ) * (1.f / 3.f) * iJ;
          float dP[3][3];
          float q = 0.f;
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const float C = cofp(Fm, Fm, r, c), dC = cofp(Fm, dF, r, c) + cofp(dF, Fm, r, c);
              dP[r][c] = da * (Fm[r][c] - bq * C) + a * (dF[r][c] - dbq * C - bq * dC);
              q = fmaf(dF[r][c], dP[r][c], q);
            }
          dea += double(q);   // v^T H_a v
          // gradH c3 H_a v: DET stores the four corners as the gradient does (three 16-byte stores; every J > 0 tet
          // contributes, so scalar stores would cost a quarter of the launch), otherwise each corner is added to hv
          // after the component's rows as soon as it is formed
          float g0[3] = {0.f, 0.f, 0.f};
          if constexpr (DET) {
            float gk[3][3];
#pragma unroll
            for (int k = 0; k < 3; ++k)
#pragma unroll
              for (int r = 0; r < 3; ++r) {
                gk[k][r] = s3 * (dP[r][0] * bb[k][0] + dP[r][1] * bb[k][1] + dP[r][2] * bb[k][2]);
                g0[r] -= gk[k][r];
              }
            det_store(tc, t, g0[0], g0[1], g0[2], gk[0][0], gk[0][1], gk[0][2], gk[1][0], gk[1][1], gk[1][2], gk[2][0], gk[2][1], gk[2][2]);
            dmask |= 1u << t;
          } else {
            wait_rows();
#pragma unroll
            for (int k = 0; k < 3; ++k) {
              const size_t vk = 3 * gid_x(tj[t][k + 1]);
#pragma unroll
              for (int r = 0; r < 3; ++r) {
                const float g = s3 * (dP[r][0] * bb[k][0] + dP[r][1] * bb[k][1] + dP[r][2] * bb[k][2]);
                g0[r] -= g;
                atomicAdd(grad + vk + r, g);
              }
            }
            const size_t v0 = 3 * gid_x(tj[t][0]);
            atomicAdd(grad + v0, g0[0]); atomicAdd(grad + v0 + 1, g0[1]); atomicAdd(grad + v0 + 2, g0[2]);
          }
        } else if (!HVP && AMIPS && amips_on && J > 0.f) {
          // AMIPS (default off; no counterpart in the reference -- SURVEY.md F1):  psi = tr(F^T F) / (3 J^(2/3)) - 1,
          // d psi / dF = 2 / (3 J^(2/3)) (F - tr / (3 J) cof F),  F = Ds B with B = Dm^-1 streamed per tet
          const int slot = lane * int(F::TPL) + t;
          const float4 *bp = p.Bt + (size_t(tcell0 + tc) * 3) * (32 * F::TPL) + slot;
          const float4 b0 = __ldg(bp), b1 = __ldg(bp + 32 * F::TPL), b2 = __ldg(bp + 64 * F::TPL);
          float Fm[3][3];
          const float ex[3] = {e1x, e2x, e3x}, ey[3] = {e1y, e2y, e3y}, ez[3] = {e1z, e2z, e3z};
          const float bb[3][3] = {{b0.x, b0.y, b0.z}, {b1.x, b1.y, b1.z}, {b2.x, b2.y, b2.z}};
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            Fm[0][c] = ex[0] * bb[0][c] + ex[1] * bb[1][c] + ex[2] * bb[2][c];
            Fm[1][c] = ey[0] * bb[0][c] + ey[1] * bb[1][c] + ey[2] * bb[2][c];
            Fm[2][c] = ez[0] * bb[0][c] + ez[1] * bb[1][c] + ez[2] * bb[2][c];
          }
          float tr = 0.f;
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) tr = fmaf(Fm[r][c], Fm[r][c], tr);
          const float cb = cbrtf(J), j23 = cb * cb;
          {
            // psi = (m - l) / l with m = tr / 3 and l = J^(2/3), formed without that difference of two values near 1 (it
            // costs about an ulp of 1 per tet, where psi is O(sigma^2) near a rotation and uniform scaling): with C = F^T F
            // and its deviator D = C - m I (tr D = 0), m^3 - l^3 = m^3 - det C = m/2 |D|^2 - det D, so psi = (m/2 |D|^2 -
            // det D) / (l (m^2 + m l + l^2)).  D's diagonal is formed from differences of C's (exact when they are close,
            // Sterbenz), so only the rounding of C enters it (DESIGN.md section 5, "Per-sphere statistics")
            float Cm[3][3];
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
              for (int j = i; j < 3; ++j) Cm[i][j] = Fm[0][i] * Fm[0][j] + Fm[1][i] * Fm[1][j] + Fm[2][i] * Fm[2][j];
            const float a01 = Cm[0][0] - Cm[1][1], a02 = Cm[0][0] - Cm[2][2], a12 = Cm[1][1] - Cm[2][2];
            const float d0 = (a01 + a02) * (1.f / 3.f), d1 = (a12 - a01) * (1.f / 3.f), d2 = -(d0 + d1);
            const float o01 = Cm[0][1], o02 = Cm[0][2], o12 = Cm[1][2];
            const float dd = fmaf(d0, d0, fmaf(d1, d1, d2 * d2)) + 2.f * fmaf(o01, o01, fmaf(o02, o02, o12 * o12));
            const float detD = d0 * (d1 * d2 - o12 * o12) - o01 * (o01 * d2 - o12 * o02) + o02 * (o01 * o12 - d1 * o02);
            const float m = tr * (1.f / 3.f);
            dea += double(fmaf(0.5f * m, dd, -detD) / (j23 * fmaf(m, m + j23, j23 * j23)));
          }
          if (grad) {
            const float a = 2.f / (3.f * j23) * s3, bq = tr / (3.f * J);
            float Pm[3][3];   // a (F - bq cof F)
            Pm[0][0] = a * (Fm[0][0] - bq * (Fm[1][1] * Fm[2][2] - Fm[1][2] * Fm[2][1]));
            Pm[0][1] = a * (Fm[0][1] - bq * (Fm[1][2] * Fm[2][0] - Fm[1][0] * Fm[2][2]));
            Pm[0][2] = a * (Fm[0][2] - bq * (Fm[1][0] * Fm[2][1] - Fm[1][1] * Fm[2][0]));
            Pm[1][0] = a * (Fm[1][0] - bq * (Fm[0][2] * Fm[2][1] - Fm[0][1] * Fm[2][2]));
            Pm[1][1] = a * (Fm[1][1] - bq * (Fm[0][0] * Fm[2][2] - Fm[0][2] * Fm[2][0]));
            Pm[1][2] = a * (Fm[1][2] - bq * (Fm[0][1] * Fm[2][0] - Fm[0][0] * Fm[2][1]));
            Pm[2][0] = a * (Fm[2][0] - bq * (Fm[0][1] * Fm[1][2] - Fm[0][2] * Fm[1][1]));
            Pm[2][1] = a * (Fm[2][1] - bq * (Fm[0][2] * Fm[1][0] - Fm[0][0] * Fm[1][2]));
            Pm[2][2] = a * (Fm[2][2] - bq * (Fm[0][0] * Fm[1][1] - Fm[0][1] * Fm[1][0]));
            if constexpr (DET) {
              float gk[3][3], g0[3] = {0.f, 0.f, 0.f};
#pragma unroll
              for (int k = 0; k < 3; ++k)
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                  gk[k][r] = Pm[r][0] * bb[k][0] + Pm[r][1] * bb[k][1] + Pm[r][2] * bb[k][2];
                  g0[r] -= gk[k][r];
                }
              det_store(tc, t, g0[0], g0[1], g0[2], gk[0][0], gk[0][1], gk[0][2], gk[1][0], gk[1][1], gk[1][2], gk[2][0], gk[2][1], gk[2][2]);
              dmask |= 1u << t;
              continue;
            }
            wait_rows();
            float g0[3] = {0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < 3; ++k) {       // vertex k+1 pulls with P a_{k+1},  a_{k+1} = row k of B
              const size_t vk = 3 * gid_x(tj[t][k + 1]);
#pragma unroll
              for (int r = 0; r < 3; ++r) {
                const float g = Pm[r][0] * bb[k][0] + Pm[r][1] * bb[k][1] + Pm[r][2] * bb[k][2];
                atomicAdd(grad + vk + r, g);
                g0[r] -= g;
              }
            }
            const size_t v0 = 3 * gid_x(tj[t][0]);
            atomicAdd(grad + v0, g0[0]); atomicAdd(grad + v0 + 1, g0[1]); atomicAdd(grad + v0 + 2, g0[2]);
          }
        }
      }
      if constexpr (LINE) {
        // warp reduce-scatter of the cell's kLN sums in fp32 (one halving per xor offset 16, 8, ...; the lanes of a pair
        // keep the upper or the lower half), then each lane adds value line_idx(lane) to its fp64 running sum
#pragma unroll
        for (int h = kLN / 2, o = 16; h >= 1; h >>= 1, o >>= 1) {
          const bool up = lane & o;
#pragma unroll
          for (int i = 0; i < h; ++i) {
            const float send = up ? lv[i] : lv[i + h], keep = up ? lv[i + h] : lv[i];
            lv[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
          }
        }
#pragma unroll
        for (int o = 16 / kLN; o >= 1; o >>= 1) lv[0] += __shfl_xor_sync(0xffffffffu, lv[0], o);
        dln += double(lv[0]);
      }
      if (DET && grad) {   // every launch with a gradient rewrites every cell's ballot: inactive slots are never read
        const unsigned m0 = __ballot_sync(0xffffffffu, dmask & 1u), m1 = F::TPL > 1 ? __ballot_sync(0xffffffffu, dmask & 2u) : 0u;
        if (lane == 0) {
          p.det_ballot[tcell0 + tc] = (static_cast<unsigned long long>(m1) << 32) | m0;
          if (m0 | m1) p.det_flag[hcur.comp] = 1u;
        }
      }
    }
    if (s == cs.x) TSB_STAMP(6);
    if (SPH && lane == 0) {
      p.sph_rec[size_t(s) * NW + warp].min_J = __int_as_float(mnK < 0 ? mnK ^ 0x7FFFFFFF : mnK);
      p.sph_rec[size_t(s) * NW + warp].n_inverted = nneg;
    }

    // ---- hand the staging buffers over ------------------------------------------------------------------
    if (s + 1 < cs.y) {      // (after the last segment the energy fold's own barrier is the only one needed)
      if (!GLOBAL) {
        const bool e2 = eager2_of();
        if (li == 0 && e2) {
          // segment 1 is already staged: no barrier
        } else {
          if (pre) {
            if (li == 1 && e2) __syncthreads();    // half 0 is reused: every warp must have left segment 0
            store_staged(hn, li + 1);
          }
          __syncthreads();
          if (!pre) {
            stage_direct(hn, li + 1);
            __syncthreads();
          }
        }
      } else if (!DET && grad) {
        __syncthreads();     // keeps the named barrier's generations apart
      }
    }
    // SPH: this warp's record of the segment (every warp writes one, also with no work in it); after the handover, so
    // that the next component's prefetch registers are no longer live
    if constexpr (SPH) {
      const double ws = warp_sum(des), wb = warp_sum(deb), wa = AMIPS ? warp_sum(dea) : 0.0;
      if (lane == 0) {
        SphRec &r = p.sph_rec[size_t(s) * NW + warp];
        r.smooth = ws; r.barrier = wb; r.amips = wa;
        red[3 * warp] += ws; red[3 * warp + 1] += wb; red[3 * warp + 2] += wa;
      }
      des = 0.0; deb = 0.0; dea = 0.0;
    }
    // LINE: the CTA's record of the segment.  The warp's values (tet value j in lane line_lane(j), then u^T M d, d^T M d
    // and the smallest root) are combined over the warps in fixed order, three per round through red[]
    if constexpr (LINE) {
      const double wud = warp_sum(deb), wmd = warp_sum(des);
      const float wmin = __uint_as_float(__reduce_min_sync(0xffffffffu, __float_as_uint(rmin)));   // roots are >= 0
      LineRec *rec = line_rec(p.sph_rec, s, NW);
      constexpr int nv = kLN + 3;
      for (int q0 = 0; q0 < nv; q0 += 3) {
        const int j = q0 + min(lane, 2);
        const double tv = __shfl_sync(0xffffffffu, dln, line_lane<kLN>(j < kLN ? j : 0));
        const double val = j < kLN ? tv : (j == kLN ? wud : (j == kLN + 1 ? wmd : double(wmin)));
        if (lane < 3 && j < nv) red[3 * warp + lane] = val;
        __syncthreads();
        if (warp == 0 && lane < 3 && j < nv) {
          double acc = red[lane];
          for (int w = 1; w < NW; ++w) acc = j == nv - 1 ? fmin(acc, red[3 * w + lane]) : acc + red[3 * w + lane];
          rec->v[j < kLN ? j : 2 * kLineMaxAlpha + (j - kLN)] = acc;
        }
        __syncthreads();
      }
      if (!AMIPS && warp == 0 && lane < kLineMaxAlpha) rec->v[kLineMaxAlpha + lane] = 0.0;
      des = 0.0; deb = 0.0; dln = 0.0;
      rmin = INFINITY;
    }
    hcur = hn;
  }
  if constexpr (!LINE) {   // LINE: no energy fold, the records are the output
    // ---- energies: lanes -> warp -> CTA partial; CTA 0 folds all partials in fixed order ---------------------
    TSB_STAMP(7);
    if constexpr (!SPH) {   // SPH: red[] already holds the warp's sums, segment by segment
      des = warp_sum(des);
      deb = warp_sum(deb);
      if (AMIPS) dea = warp_sum(dea);
      if (lane == 0) { red[3 * warp] = des; red[3 * warp + 1] = deb; red[3 * warp + 2] = dea; }
    }
    __syncthreads();
    TSB_STAMP(8);
    if (tid == 0) {
      double a = 0.0, b = 0.0, c = 0.0;
      for (int w = 0; w < NW; ++w) { a += red[3 * w]; b += red[3 * w + 1]; c += red[3 * w + 2]; }
      if constexpr (!HVP) a *= 0.5;   // HVP: v^T M v itself
      // two 16-byte stores carry the partials; their arrival IS the "this CTA is done" signal (no fence, no ticket)
      unsigned long long ua = (unsigned long long)__double_as_longlong(a), ub = (unsigned long long)__double_as_longlong(b);
      unsigned long long uc = (unsigned long long)__double_as_longlong(c);
      if (ua == kSentinel) ua = 0x7FF8000000000000ull;
      if (ub == kSentinel) ub = 0x7FF8000000000000ull;
      if (uc == kSentinel) uc = 0x7FF8000000000000ull;
      asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(p.cta_energy + 4 * blockIdx.x), "l"(ua), "l"(ub) : "memory");
      asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(p.cta_energy + 4 * blockIdx.x + 2), "l"(uc), "l"(0ull) : "memory");
    }
    TSB_STAMP(9);
    if (blockIdx.x == 0 && warp == 0) {
      __syncwarp();
      double a = 0.0, b = 0.0, c3sum = 0.0;
      // Each lane owns slots lane, lane + 32, ...; the loads of a batch of kPollBatch slots are issued together, so one
      // L2 round trip after the last partial has landed finishes the fold (polling them one after the other cost five
      // dependent round trips, ~2 us per launch).  The summation order stays fixed: slot order per lane, then the shuffle tree.
      constexpr int kPollBatch = 5;
      for (int c0 = lane; c0 < int(gridDim.x); c0 += 32 * kPollBatch) {
        unsigned long long ua[kPollBatch], ub[kPollBatch], uc[kPollBatch], ud[kPollBatch];
        bool pending = true;
        while (pending) {
          pending = false;
#pragma unroll
          for (int k = 0; k < kPollBatch; ++k) {
            const int c = c0 + 32 * k;
            if (c < int(gridDim.x)) {
              asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(ua[k]), "=l"(ub[k]) : "l"(p.cta_energy + 4 * c) : "memory");
              asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(uc[k]), "=l"(ud[k]) : "l"(p.cta_energy + 4 * c + 2) : "memory");
            }
          }
#pragma unroll
          for (int k = 0; k < kPollBatch; ++k)
            if (c0 + 32 * k < int(gridDim.x)) pending |= ua[k] == kSentinel || ub[k] == kSentinel || uc[k] == kSentinel || ud[k] == kSentinel;
        }
#pragma unroll
        for (int k = 0; k < kPollBatch; ++k) {
          const int c = c0 + 32 * k;
          if (c < int(gridDim.x)) {
            asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(p.cta_energy + 4 * c), "l"(kSentinel), "l"(kSentinel) : "memory");   // re-arm
            asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(p.cta_energy + 4 * c + 2), "l"(kSentinel), "l"(kSentinel) : "memory");
            a += __longlong_as_double((long long)ua[k]);
            b += __longlong_as_double((long long)ub[k]);
            c3sum += __longlong_as_double((long long)uc[k]);
          }
        }
      }
      a = warp_sum(a); b = warp_sum(b); c3sum = warp_sum(c3sum);
      if (lane == 0 && (!(HVP || DIAG) || p.energy_out)) {   // HVP: energy_out is the optional curvature; DIAG: nullptr
        p.energy_out[0] = float(double(p.c1) * a + double(p.c2) * b + double(p.c3) * c3sum);
        p.energy_out[1] = float(a);
        p.energy_out[2] = float(b);
        if (p.energy4) p.energy_out[3] = float(c3sum);
      }
      if (!DET)
        for (int c = lane; c < p.n_components; c += 32) p.done[c] = 0u;   // every CTA has finished: safe to re-arm
    }
    TSB_STAMP(10);
  }
#ifdef TSB_TRACE
  if (tid == 0 && p.trace) p.trace[blockIdx.x * kTraceSlots + 11] = gtime();
#endif
}

// GLOBAL mode pre-pass: u = rel_u(x, X, c), c = fp32(x_r - X_r) of the component's reference vertex r = X4[v].w (see
// staging_tables in tsb_plan.cpp), and x as float4 per vertex.
__global__ void prestage_kernel(const float *__restrict__ x, const float4 *__restrict__ X4, float4 *__restrict__ u4,
                                float4 *__restrict__ x4, int n) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    const float4 X = X4[v];
    const size_t r = size_t(__float_as_uint(X.w));
    const float4 Xr = X4[r];
    const float a = x[3 * size_t(v)], b = x[3 * size_t(v) + 1], c = x[3 * size_t(v) + 2];
    const float c0 = x[3 * r] - Xr.x, c1 = x[3 * r + 1] - Xr.y, c2 = x[3 * r + 2] - Xr.z;
    u4[v] = make_float4(rel_u(a, X.x, c0), rel_u(b, X.y, c1), rel_u(c, X.z, c2), 0.f);
    x4[v] = make_float4(a, b, c, 0.f);
  }
}

// The same for the HVP instantiation: u = v - v_r with r = X4[v].w, and x as float4 per vertex.
__global__ void prestage_hvp_kernel(const float *__restrict__ x, const float *__restrict__ dir, const float4 *__restrict__ X4,
                                    float4 *__restrict__ u4, float4 *__restrict__ x4, int n) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    const size_t r = size_t(__float_as_uint(X4[v].w));
    u4[v] = make_float4(dir[3 * size_t(v)] - dir[3 * r], dir[3 * size_t(v) + 1] - dir[3 * r + 1], dir[3 * size_t(v) + 2] - dir[3 * r + 2], 0.f);
    x4[v] = make_float4(x[3 * size_t(v)], x[3 * size_t(v) + 1], x[3 * size_t(v) + 2], 0.f);
  }
}

// Deterministic gather, after a DET launch on the same stream: CTA = a run of <= kDetChunkRows vertex rows of one
// component (thread = row).  Unflagged components are skipped without reading their lists.  A row sums the corner
// vectors of its list's active entries in list order, starting from +0, and adds the sum to grad: it is the only
// writer of its row, so the result does not depend on scheduling.  The last CTA of a flagged component to finish
// clears the flag (flag = 1 + number of CTAs done, so every CTA reads it before it is cleared).
__global__ void __launch_bounds__(kDetChunkRows) det_gather_kernel(const DetParams d, float *__restrict__ grad) {
  asm volatile("griddepcontrol.wait;" ::: "memory");       // everything below reads what the energy kernel wrote
                                                             // (a no-op under the plain launch used now)
  const int2 ch = __ldg(&d.chunk[blockIdx.x]);               // (component, first row)
  const unsigned flag = __ldcg(d.flag + ch.x);
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (!flag) return;
  const int row0 = __ldg(&d.comp_row[ch.x]), row_end = __ldg(&d.comp_row[ch.x + 1]);
  const int r = ch.y + int(threadIdx.x);
  if (r < row_end) {
    const int b = __ldg(&d.rowptr[r]), e = __ldg(&d.rowptr[r + 1]);
    const float *sc = reinterpret_cast<const float *>(d.scratch);
    const uint32_t tpl_mask = (1u << d.tpl_log) - 1u, cell_log = 5 + d.tpl_log;
    float ax = 0.f, ay = 0.f, az = 0.f;
    bool any = false;
#pragma unroll 4
    for (int i = b; i < e; ++i) {
      const uint32_t ent = __ldg(&d.ent[i]), slot = ent >> 2, k = ent & 3u;
      const uint32_t sic = slot & ((1u << cell_log) - 1u);                  // lane * TPL + t
      const unsigned long long m = __ldcg(d.ballot + (slot >> cell_log));
      const bool act = (m >> (((sic & tpl_mask) << 5) | (sic >> d.tpl_log))) & 1ull;
      // inactive slots hold stale values: loaded anyway (no dependence on the ballot), never added
      const float *c = sc + size_t(slot) * 12 + k * 3;
      const float cx = __ldcg(c), cy = __ldcg(c + 1), cz = __ldcg(c + 2);
      if (act) { ax += cx; ay += cy; az += cz; any = true; }
    }
    if (any) {
      const size_t v = 3 * size_t(__ldg(&d.vert[r]));
      grad[v] += ax; grad[v + 1] += ay; grad[v + 2] += az;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned nchunks = unsigned((row_end - row0 + kDetChunkRows - 1) / kDetChunkRows);
    if (nchunks == 1 || atomicAdd(d.flag + ch.x, 1u) == nchunks) d.flag[ch.x] = 0u;
  }
}

// Per-sphere statistics, after an SPH launch on the same stream: one warp per component.  Lane l sums the component's
// (segment, warp) records l, l + 32, ... in that order, a shuffle tree combines the lanes: the result depends on the
// records alone, never on scheduling.  Every output record is rewritten.
constexpr int kFoldWarps = 8;
__global__ void __launch_bounds__(kFoldWarps * 32) sphere_fold_kernel(const SphParams sp, tsb_sphere_stats_t *__restrict__ out) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the next energy launch writes records only after its wait
  const int c = blockIdx.x * kFoldWarps + int(threadIdx.x >> 5), lane = int(threadIdx.x & 31);
  if (c >= sp.n_components) return;
  const int r0 = __ldg(&sp.comp_seg[c]) * sp.nw, r1 = __ldg(&sp.comp_seg[c + 1]) * sp.nw;
  double a = 0.0, b = 0.0, d = 0.0;
  float m = INFINITY;
  int k = 0;
  for (int r = r0 + lane; r < r1; r += 32) {
    const SphRec e = sp.rec[r];
    a += e.smooth; b += e.barrier; d += e.amips;
    m = fminf(m, e.min_J);
    k += e.n_inverted;
  }
  a = warp_sum(a); b = warp_sum(b); d = warp_sum(d);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  k = __reduce_add_sync(0xffffffffu, k);
  if (lane == 0) {
    tsb_sphere_stats_t r;
    r.smooth = 0.5 * a;            // as the CTA fold: 1/2 u^T M u
    r.barrier = b;
    r.amips = d;
    r.min_J = m;
    r.n_inverted = k;
    r.n_tets = __ldg(&sp.comp_ntets[c]);
    r.first_vertex = __ldg(&sp.comp_first_vertex[c]);
    out[c] = r;
  }
}

// Line search, after a LINE launch on the same stream.  Every sum below runs in a fixed order over the records alone.
struct LineArgs {
  const float *alpha;
  int32_t n_alpha;
  float c1, c2, c3;
};

// (c1 ds + c2 db + c3 da, ds, db, da) at alpha_k from a (component or total) value set held one value per lane (lane j:
// value j of LineRec), written by lane k < n_alpha to out[4k..4k+3]; ds = alpha u^T M d + 1/2 alpha^2 d^T M d
__device__ __forceinline__ void line_write_delta(double v, int lane, const LineArgs &la, float *out) {
  const double ud = __shfl_sync(0xffffffffu, v, 2 * kLineMaxAlpha), dd = __shfl_sync(0xffffffffu, v, 2 * kLineMaxAlpha + 1);
  const double db = __shfl_sync(0xffffffffu, v, lane & (kLineMaxAlpha - 1));
  const double da = __shfl_sync(0xffffffffu, v, kLineMaxAlpha + (lane & (kLineMaxAlpha - 1)));
  if (out && lane < la.n_alpha) {
    const double al = double(__ldg(la.alpha + lane));
    const double ds = al * ud + 0.5 * (al * al) * dd;
    out[4 * lane] = float(double(la.c1) * ds + double(la.c2) * db + double(la.c3) * da);
    out[4 * lane + 1] = float(ds);
    out[4 * lane + 2] = float(db);
    out[4 * lane + 3] = float(da);
  }
}

// One warp per component: lane j < kLineVals folds value j of the component's segment records in segment order (the
// root: their minimum) and stores it over the record of the component's first segment (each lane reads and writes its
// own slot only), then the optional per-sphere outputs.
__global__ void __launch_bounds__(kFoldWarps * 32) line_fold_kernel(const SphParams sp, const LineArgs la, float *__restrict__ sd,
                                                                    float *__restrict__ ss) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int c = blockIdx.x * kFoldWarps + int(threadIdx.x >> 5), lane = int(threadIdx.x & 31);
  if (c >= sp.n_components) return;
  SphRec *rec = const_cast<SphRec *>(sp.rec);
  const int s0 = __ldg(&sp.comp_seg[c]), s1 = __ldg(&sp.comp_seg[c + 1]);
  double v = 0.0;
  if (lane < kLineVals) {
    v = line_rec(rec, s0, sp.nw)->v[lane];
    for (int s = s0 + 1; s < s1; ++s) {
      const double e = line_rec(rec, s, sp.nw)->v[lane];
      v = lane == kLineVals - 1 ? fmin(v, e) : v + e;
    }
    line_rec(rec, s0, sp.nw)->v[lane] = v;
  }
  line_write_delta(v, lane, la, sd ? sd + size_t(c) * la.n_alpha * 4 : nullptr);
  if (ss && lane == kLineVals - 1) ss[c] = float(v);
}

// One CTA: warp w folds the components w, w + kFoldWarps, ... in order (lane j: value j), warp 0 the warps' partials in
// order; then delta_out and step_out.
__global__ void __launch_bounds__(kFoldWarps * 32) line_total_kernel(const SphParams sp, const LineArgs la, float *__restrict__ delta,
                                                                     float *__restrict__ step) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  __shared__ double part[kFoldWarps][kLineVals];
  const int w = int(threadIdx.x >> 5), lane = int(threadIdx.x & 31);
  const SphRec *rec = sp.rec;
  if (lane < kLineVals) {
    double v = lane == kLineVals - 1 ? double(INFINITY) : 0.0;
    for (int c = w; c < sp.n_components; c += kFoldWarps) {
      const double e = line_rec(const_cast<SphRec *>(rec), __ldg(&sp.comp_seg[c]), sp.nw)->v[lane];
      v = lane == kLineVals - 1 ? fmin(v, e) : v + e;
    }
    part[w][lane] = v;
  }
  __syncthreads();
  if (w != 0) return;
  double v = 0.0;
  if (lane < kLineVals) {
    v = part[0][lane];
    for (int k = 1; k < kFoldWarps; ++k) v = lane == kLineVals - 1 ? fmin(v, part[k][lane]) : v + part[k][lane];
  }
  line_write_delta(v, lane, la, delta);
  if (step && lane == kLineVals - 1) step[0] = float(v);
}

// ---- level-1 helpers -------------------------------------------------------------------------------
__global__ void scale_kernel(const float *__restrict__ g, int64_t count, float gradH, const float *gradH_dev,
                             float *__restrict__ out) {
  const float s = gradH * (gradH_dev ? __ldg(gradH_dev) : 1.f);
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < count; i += int64_t(gridDim.x) * blockDim.x)
    out[i] = s * g[i];
}

__device__ __forceinline__ void block_max_to(float v, float *dst) {
  // v >= 0.  Order-preserving uint compare for non-negative floats.
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __shared__ float s_m[32];
  if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    float m = (threadIdx.x < (blockDim.x + 31) / 32) ? s_m[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) atomicMax(reinterpret_cast<unsigned int *>(dst), __float_as_uint(m));
  }
  __syncthreads();
}

__global__ void absmax_kernel(const float *__restrict__ g, int64_t count, float *work) {
  float m = 0.f;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < count; i += int64_t(gridDim.x) * blockDim.x)
    m = fmaxf(m, fabsf(g[i]));
  block_max_to(m, work);
}

// if max|g| > thr: g *= s / max|g|.  Consumes and re-zeroes work[0] through a ticket in work[1].
__global__ void grad_limit_apply_kernel(float *g, int64_t count, float thr, float s, float *work) {
  const float m = __ldcg(work);
  if (m > thr) {
    const float f = s / m;
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < count; i += int64_t(gridDim.x) * blockDim.x) g[i] *= f;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int *ticket = reinterpret_cast<unsigned int *>(work + 1);
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) { work[0] = 0.f; *ticket = 0u; }
  }
}

// AdamUniform (utils/optimizer.py:37-89), pass 1: moments + the two global maxima.
__global__ void adam_uniform_moments_kernel(const float *__restrict__ grad, float *__restrict__ g1, float *__restrict__ g2,
                                            int64_t count, float b1, float b2, float omb1, float omb2, float inv_bc1,
                                            float inv_bc2, float *work) {
  float mx2 = 0.f, mx1 = 0.f;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < count; i += int64_t(gridDim.x) * blockDim.x) {
    const float g = grad[i];
    const float m1 = b1 * g1[i] + omb1 * g;                 // optimizer.py:61  (1 - beta formed in double on the host, like Python)
    const float m2 = b2 * g2[i] + omb2 * (g * g);           // optimizer.py:62
    g1[i] = m1; g2[i] = m2;
    mx2 = fmaxf(mx2, sqrtf(m2 * inv_bc2));                  // optimizer.py:68,74
    mx1 = fmaxf(mx1, fabsf(m1 * inv_bc1));                  // optimizer.py:67,83
  }
  block_max_to(mx2, work);
  block_max_to(mx1, work + 1);
}

// pass 2: p -= lr * clamp(m1_hat / (1e-8 + max sqrt(m2_hat)))   (optimizer.py:74-88)
__global__ void adam_uniform_apply_kernel(float *__restrict__ p, const float *__restrict__ g1, int64_t count, float lr,
                                          float inv_bc1, float grad_limit, float *work, unsigned int *ticket) {
  const float denom = 1e-8f + __ldcg(work);
  float f = inv_bc1 / denom;
  if (grad_limit > 0.f) {
    const float s = __ldcg(work + 1) / denom;               // max |gr|
    if (s > grad_limit) f *= grad_limit / s;
  }
  f *= lr;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < count; i += int64_t(gridDim.x) * blockDim.x) p[i] -= f * g1[i];
  __syncthreads();
  if (threadIdx.x == 0) {
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) { work[0] = 0.f; work[1] = 0.f; *ticket = 0u; }
  }
}

inline int grid_for(int64_t count, int block) {
  constexpr int64_t kMaxGrid = 132 * 8;     // 8 resident 256-thread CTAs on each of an H100 SXM's 132 SMs
  int64_t g = (count + block - 1) / block;
  return int(g < 1 ? 1 : (g > kMaxGrid ? kMaxGrid : g));
}

// ---- the energy_grad_kernel instantiations, by flag bits f = AMIPS | DET << 1 | SPH << 2 | HVP << 3 | LINE << 4 |
// DIAG << 5 ------------------------------------------------------------------------------------------------------------
using EnergyKernel = void (*)(KParams);

// HVP is never combined with SPH, LINE with nothing but AMIPS, DIAG with nothing but AMIPS and DET: those entries are
// nullptr and never instantiated
template <int NW, int MINB, bool GLOBAL, int F>
constexpr EnergyKernel kernel_of() {
  if constexpr ((F & 8) && (F & 4)) return nullptr;
  else if constexpr ((F & 16) && (F & 14)) return nullptr;
  else if constexpr ((F & 32) && (F & 28)) return nullptr;
  else if constexpr (F & 32) return energy_grad_kernel<NW, MINB, GLOBAL, bool(F & 1), bool(F & 2), false, false, false, true>;
  else if constexpr (F & 16) return energy_grad_kernel<NW, MINB, GLOBAL, bool(F & 1), false, false, false, true>;
  else return energy_grad_kernel<NW, MINB, GLOBAL, bool(F & 1), bool(F & 2), bool(F & 4), bool(F & 8)>;
}

template <int NW, int MINB, bool GLOBAL, int... F>
const EnergyKernel *flag_table(std::integer_sequence<int, F...>) {
  static const EnergyKernel table[] = {kernel_of<NW, MINB, GLOBAL, F>()...};
  return table;
}

// 16 warps run one CTA per SM, 8 warps two; nullptr for any other nw or a combination that is not instantiated
EnergyKernel energy_kernel(int nw, bool global, bool amips, bool det, bool sph, bool hvp = false, bool line = false,
                           bool diag = false) {
  constexpr std::make_integer_sequence<int, 64> flags{};
  const int f = int(amips) | int(det) << 1 | int(sph) << 2 | int(hvp) << 3 | int(line) << 4 | int(diag) << 5;
  if (nw == 16) return (global ? flag_table<16, 1, true>(flags) : flag_table<16, 1, false>(flags))[f];
  if (nw == 8) return (global ? flag_table<8, 2, true>(flags) : flag_table<8, 2, false>(flags))[f];
  return nullptr;
}

}  // namespace

int energy_ring_bytes(int slots, int cells_per_chunk, bool global) { return slots * cells_per_chunk * (global ? kCellGlobal : kCellStaged); }

int energy_smem_bytes(int nw, int ring_slots, int cells_per_chunk, int area_verts, bool global) {
  return smem_total(global ? 0 : area_verts * 32, nw, energy_ring_bytes(ring_slots, cells_per_chunk, global));
}

cudaError_t energy_occupancy(int nw, int smem_bytes, bool global, bool amips, bool det, int *ctas_per_sm) {
  if (!energy_kernel(nw, global, false, false, false)) return cudaErrorInvalidValue;
  // opt in to the device maximum (the attribute is per function, not per handle: handles with different staging sizes
  // share the kernel)
  int dev = 0, optin = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e != cudaSuccess) return e;
  *ctas_per_sm = 0;
  if (smem_bytes > optin) return cudaSuccess;   // does not fit
  // every instantiation the handle may launch: AMIPS ones when amips, DET ones when det, with and without SPH, and the
  // HVP ones (tsb_hvp, and tsb_hvp_ex's AMIPS ones when amips), the LINE ones (tsb_line_search) and the DIAG ones
  // (tsb_hess_diag)
  int ctas = 1 << 30;
  for (int f = 0; f < 64; ++f) {
    if (((f & 1) && !amips) || ((f & 2) && !det)) continue;
    const EnergyKernel k = energy_kernel(nw, global, f & 1, f & 2, f & 4, f & 8, f & 16, f & 32);
    if (!k) continue;   // HVP with SPH, LINE with anything but AMIPS, DIAG with anything but AMIPS and DET
    if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, optin) != cudaSuccess) {
      cudaGetLastError();
      return cudaSuccess;   // does not fit
    }
    int c = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, k, nw * 32, size_t(smem_bytes));
    if (e != cudaSuccess) return e;
    ctas = std::min(ctas, c);
  }
  *ctas_per_sm = ctas;
  return cudaSuccess;
}

cudaError_t launch_energy_grad(const KParams &p, const LaunchConfig &lc, cudaStream_t stream) {
  const EnergyKernel k = energy_kernel(lc.nw, lc.global, lc.amips, lc.det, lc.sph, lc.hvp, lc.line, lc.diag);
  if (!k) return cudaErrorInvalidValue;
  if (lc.global) {
    if (lc.hvp || lc.line) prestage_hvp_kernel<<<grid_for(p.n, 256), 256, 0, stream>>>(p.x, p.v, p.X4, p.u4g, p.x4g, p.n);
    else prestage_kernel<<<grid_for(p.n, 256), 256, 0, stream>>>(p.x, p.X4, p.u4g, p.x4g, p.n);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(unsigned(lc.grid));
  cfg.blockDim = dim3(unsigned(lc.nw * 32));
  cfg.dynamicSmemBytes = size_t(lc.smem_bytes);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, k, p);
}

// A plain launch (the gather starts when the energy kernel has finished); its early launch_dependents still lets the
// next energy launch start its plan prefetch while the gather runs.  Launching the gather with programmatic dependent
// launch as well measured 5x slower at 64 x 4096 with inverted tets (DESIGN.md section 3).
cudaError_t launch_det_gather(const DetParams &d, float *grad, cudaStream_t stream) {
  det_gather_kernel<<<unsigned(d.n_chunks), kDetChunkRows, 0, stream>>>(d, grad);
  return cudaGetLastError();
}

cudaError_t launch_sphere_fold(const SphParams &sp, tsb_sphere_stats_t *out, cudaStream_t stream) {
  sphere_fold_kernel<<<unsigned((sp.n_components + kFoldWarps - 1) / kFoldWarps), kFoldWarps * 32, 0, stream>>>(sp, out);
  return cudaGetLastError();
}

cudaError_t launch_line_fold(const SphParams &sp, const float *alpha, int n_alpha, float c1, float c2, float c3,
                             float *delta_out, float *step_out, float *sphere_delta_out, float *sphere_step_out,
                             cudaStream_t stream) {
  const LineArgs la{alpha, n_alpha, c1, c2, c3};
  if (sp.n_components > 0)
    line_fold_kernel<<<unsigned((sp.n_components + kFoldWarps - 1) / kFoldWarps), kFoldWarps * 32, 0, stream>>>(
        sp, la, sphere_delta_out, sphere_step_out);
  line_total_kernel<<<1, kFoldWarps * 32, 0, stream>>>(sp, la, delta_out, step_out);
  return cudaGetLastError();
}

cudaError_t launch_scale(const float *g, int64_t count, float gradH, const float *gradH_dev, float *out, cudaStream_t s) {
  scale_kernel<<<grid_for(count, 256), 256, 0, s>>>(g, count, gradH, gradH_dev, out);
  return cudaGetLastError();
}

cudaError_t launch_grad_limit(float *g, int64_t count, float thr, float s, float *work4, cudaStream_t st) {
  const int grid = grid_for(count, 256);
  absmax_kernel<<<grid, 256, 0, st>>>(g, count, work4);
  grad_limit_apply_kernel<<<grid, 256, 0, st>>>(g, count, thr, s, work4);
  return cudaGetLastError();
}

cudaError_t launch_adam_uniform(float *p, const float *grad, float *g1, float *g2, int64_t count, double lr, double b1,
                                double b2, int step, double grad_limit, float *work, cudaStream_t st) {
  const float inv_bc1 = float(1.0 / (1.0 - pow(b1, double(step))));   // optimizer.py:67
  const float inv_bc2 = float(1.0 / (1.0 - pow(b2, double(step))));   // optimizer.py:68
  const int grid = grid_for(count, 256);
  adam_uniform_moments_kernel<<<grid, 256, 0, st>>>(grad, g1, g2, count, float(b1), float(b2), float(1.0 - b1), float(1.0 - b2),
                                                    inv_bc1, inv_bc2, work);
  adam_uniform_apply_kernel<<<grid, 256, 0, st>>>(p, g1, count, float(lr), inv_bc1, float(grad_limit), work,
                                                  reinterpret_cast<unsigned int *>(work + 2));
  return cudaGetLastError();
}

}  // namespace tsb
