// Fused geometry-energy + gradient kernel for sm_90a (H100), plus the small level-1 helpers.
//
// ONE launch replaces the reference's forward+backward pipeline
// (tssplat_ext/tet_spheres/tet_spheres_cuda.cu:118-263: SpMV GTLTLG.x, Sdot, SpMV G.x,
// cuda_forward_det, Sasum, SpMV c1.GTLTLG.x, SpMV G.x again, cuda_backward_det, SpMV G^T, Sscal,
// with three host syncs).
//
// Math (DESIGN.md section 3).  With u = x - X (X = rest positions):
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
// ring with TMA bulk copies (cp.async.bulk + mbarrier complete_tx), issued by its lane 0, first
// chunks before griddepcontrol.wait: plan data streams from HBM while the previous kernel drains.
// Per segment the CTA stages u and x of the whole component in shared memory (float4 each; the next
// component is prefetched through registers), so all gathers are LDS.128.  Energies: per-lane fp64
// partials -> per-CTA pair -> last-arriving CTA folds them in fixed order (deterministic).
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

#include "tsb_kernels.cuh"

namespace tsb {

namespace {

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
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

// Profiling build only (-DTSB_TRACE, tools/trace_phases.py): thread 0 of every CTA stamps its phases.
#ifdef TSB_TRACE
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define TSB_STAMP(i) do { if (tid == 0 && p.trace) p.trace[blockIdx.x * 16 + (i)] = (i) == 0 ? gtime() : (unsigned long long)clock64(); } while (0)
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
    }
  }
};

template <int NW, int MINB, bool GLOBAL, bool AMIPS>
__global__ void __launch_bounds__(NW * 32, MINB) energy_grad_kernel(const KParams p) {
  using F = Fmt<GLOBAL>;
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
    ws.cell = ws.ring;
    ws.cc = 0; ws.slot = 0; ws.phase = 0; ws.lane = lane;
    if (lane == 0) {
      for (uint32_t i = 0; i < ws.nslot; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(ws.bars + i * 8), "r"(1) : "memory");
      mbar_fence_init();
      for (uint32_t i = 0; i < ws.nslot && ws.bytes_left; ++i) ws.request(smem_u32(ws.ring) + i * ws.chunk_bytes, ws.bars + i * 8);
    }
    __syncwarp();
  }
  const int vh = p.vh;
  // float4 index of a segment's u / x arrays inside the staging area (must match tsb_plan.cpp)
  auto ubase_of = [&](const SegHdr &h, int li) -> int { return h.whole ? 0 : (li & 1) * 2 * vh; };
  auto xbase_of = [&](const SegHdr &h, int li) -> int { return h.whole ? h.npos : (li & 1) * 2 * vh + vh; };

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
    if (!GLOBAL && !hcur.whole) {   // rest positions of the first component: plan data, loaded before the wait
#pragma unroll
      for (int k = 0; k < SV; ++k) {
        const int v = tid + k * NT;
        if (v < hcur.nv) { pX[k] = __ldg(&p.X4[hcur.x4off + v]); pX[k].w = __uint_as_float(uint32_t(__ldg(&p.pos16[hcur.x4off + v]))); }
      }
    }
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
    }
  }

  double des = 0.0, deb = 0.0, dea = 0.0;     // per-lane energy partials (smoothness, barrier, AMIPS)

  auto load_x = [&](const SegHdr &h) {      // x of a double-buffered component -> registers
#pragma unroll
    for (int k = 0; k < SV; ++k) {
      const int v = tid + k * NT;
      if (v < h.nv) {
        const size_t gi = size_t(h.vbase >= 0 ? h.vbase + v : __ldg(&p.vlist[h.x4off + v]));
        px[k][0] = __ldcg(p.x + 3 * gi); px[k][1] = __ldcg(p.x + 3 * gi + 1); px[k][2] = __ldcg(p.x + 3 * gi + 2);
      }
    }
  };
  auto store_staged = [&](const SegHdr &h, int li) {
    float4 *ub = stage + ubase_of(h, li), *xb = stage + xbase_of(h, li);
#pragma unroll
    for (int k = 0; k < SV; ++k) {
      const int v = tid + k * NT;
      if (v < h.nv) {
        const uint32_t pos = __float_as_uint(pX[k].w);
        ub[pos] = make_float4(px[k][0] - pX[k].x, px[k][1] - pX[k].y, px[k][2] - pX[k].z, 0.f);
        xb[pos] = make_float4(px[k][0], px[k][1], px[k][2], 0.f);
      }
    }
  };
  auto stage_direct = [&](const SegHdr &h, int li) {   // any size, no register prefetch
    float4 *ub = stage + ubase_of(h, li), *xb = stage + xbase_of(h, li);
    for (int v = tid; v < h.nv; v += NT) {
      const float4 X = __ldg(&p.X4[h.x4off + v]);
      const size_t gi = size_t(h.vbase >= 0 ? h.vbase + v : __ldg(&p.vlist[h.x4off + v]));
      const float x0 = __ldcg(p.x + 3 * gi), x1 = __ldcg(p.x + 3 * gi + 1), x2 = __ldcg(p.x + 3 * gi + 2);
      const uint32_t pos = __ldg(&p.pos16[h.x4off + v]);
      ub[pos] = make_float4(x0 - X.x, x1 - X.y, x2 - X.z, 0.f);
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
      } else if (!eager2) {
        load_x(hcur); store_staged(hcur, 0);
      } else {
        // both components' loads in flight together (second register set), then both stores
        float qx[SV][3];
        float4 qX[SV];
#pragma unroll
        for (int k = 0; k < SV; ++k) {
          const int v = tid + k * NT;
          if (v < h1.nv) { qX[k] = __ldg(&p.X4[h1.x4off + v]); qX[k].w = __uint_as_float(uint32_t(__ldg(&p.pos16[h1.x4off + v]))); }
        }
        load_x(hcur);
#pragma unroll
        for (int k = 0; k < SV; ++k) {
          const int v = tid + k * NT;
          if (v < h1.nv) {
            const size_t gi = size_t(h1.vbase >= 0 ? h1.vbase + v : __ldg(&p.vlist[h1.x4off + v]));
            qx[k][0] = __ldcg(p.x + 3 * gi); qx[k][1] = __ldcg(p.x + 3 * gi + 1); qx[k][2] = __ldcg(p.x + 3 * gi + 2);
          }
        }
        store_staged(hcur, 0);
        float4 *ub = stage + ubase_of(h1, 1), *xb = stage + xbase_of(h1, 1);
#pragma unroll
        for (int k = 0; k < SV; ++k) {
          const int v = tid + k * NT;
          if (v < h1.nv) {
            const uint32_t pos = __float_as_uint(qX[k].w);
            ub[pos] = make_float4(qx[k][0] - qX[k].x, qx[k][1] - qX[k].y, qx[k][2] - qX[k].z, 0.f);
            xb[pos] = make_float4(qx[k][0], qx[k][1], qx[k][2], 0.f);
          }
        }
      }
    }
    __syncthreads();
    TSB_STAMP(4);
  } else {
    __syncthreads();      // segment tables visible
  }
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
        pre = !hcur.whole && !hn.whole && !(li == 0 && eager2);
        if (pre) {
#pragma unroll
          for (int k = 0; k < SV; ++k) {
            const int v = tid + k * NT;
            if (v < hn.nv) { pX[k] = __ldg(&p.X4[hn.x4off + v]); pX[k].w = __uint_as_float(uint32_t(__ldg(&p.pos16[hn.x4off + v]))); }
          }
          load_x(hn);
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
    // reference displacement of the component: sum_i g_i = 0, so 1/2 sum_i (u_i - uref).g_i is the same
    // energy with the rigid translation taken out of the cancellation
    const float4 uref = GLOBAL ? __ldg(p.u4g + hcur.x4off) : stage[ubase_of(hcur, li)];
    if (s == cs.x) TSB_STAMP(13);

    // ---- operator rows: L lanes per vertex row (header in slot 0 of the first quad) ------------------
    for (int rb = 0; rb < int(wseg.x); ++rb) {
      const uint32_t hdr = *reinterpret_cast<const uint32_t *>(ws.cell + WOFF + lane * 16);
      const uint32_t rid = hdr & 0xFFFFFFu, len4 = (hdr >> 24) & 63u, llog = hdr >> 30;   // global row id | quads | log2(lanes per row)
      const bool active = rid != 0xFFFFFFu;
      const uint32_t rowj = GLOBAL ? *reinterpret_cast<const uint32_t *>(ws.cell + lane * 16)
                                   : uint32_t(*reinterpret_cast<const uint16_t *>(ws.cell + lane * 8));
      const float4 ui = gatherU(rowj);
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
      if (s == cs.x && rb == 0) { TSB_STAMP(14); if (tid == 0 && p.trace) p.trace[blockIdx.x * 16 + 15] = len4 | (uint32_t(wseg.x) << 16) | (uint32_t(wseg.y) << 24); }
#endif
      float ax = sum2(AX), ay = sum2(AY), az = sum2(AZ);
      for (uint32_t o = 1; o < (1u << llog); o <<= 1) {   // the L lanes of a row are adjacent
        ax += __shfl_xor_sync(0xffffffffu, ax, o);
        ay += __shfl_xor_sync(0xffffffffu, ay, o);
        az += __shfl_xor_sync(0xffffffffu, az, o);
      }
      if (active && (lane & ((1u << llog) - 1u)) == 0) {
        des += double(fmaf(ui.x - uref.x, ax, fmaf(ui.y - uref.y, ay, (ui.z - uref.z) * az)));
        if (grad) {
          const size_t gi = rid;
          grad[3 * gi] = s1 * ax; grad[3 * gi + 1] = s1 * ay; grad[3 * gi + 2] = s1 * az;
        }
      }
    }
    if (s == cs.x) TSB_STAMP(5);
    if (grad) {   // all warps' rows of this segment are stored -> ONE release of the component's counter, sent by
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
    const int tcell0 = amips_on ? __ldg(&p.wtc0[size_t(s) * NW + warp]) : 0;
    for (int tc = 0; tc < int(wseg.y); ++tc) {
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
      float4 xv[F::TPL][4];
#pragma unroll
      for (int t = 0; t < int(F::TPL); ++t)
#pragma unroll
        for (int k = 0; k < 4; ++k) xv[t][k] = gatherX(tj[t][k]);
      ws.advance(1);
#pragma unroll
      for (int t = 0; t < int(F::TPL); ++t) {
        const float4 x0 = xv[t][0], x1 = xv[t][1], x2 = xv[t][2], x3 = xv[t][3];
        const float idet = tdet[t];
        const float e1x = x1.x - x0.x, e1y = x1.y - x0.y, e1z = x1.z - x0.z;
        const float e2x = x2.x - x0.x, e2y = x2.y - x0.y, e2z = x2.z - x0.z;
        const float e3x = x3.x - x0.x, e3y = x3.y - x0.y, e3z = x3.z - x0.z;
        const float c1x = e2y * e3z - e2z * e3y, c1y = e2z * e3x - e2x * e3z, c1z = e2x * e3y - e2y * e3x;   // e2 x e3
        const float J = (e1x * c1x + e1y * c1y + e1z * c1z) * idet;
        if (J < 0.f) {
          const float m = -J, m2 = m * m;
          deb += double(order2 ? m2 : m2 * m2);
          if (grad) {
            const float coef = order2 ? 2.f * m : 4.f * m2 * m;       // p (-J)^(p-1)
            const float k = -coef * idet * s2;                         // gradH c2 dphi/dJ / det(Dm)
            const float g1x = k * c1x, g1y = k * c1y, g1z = k * c1z;
            const float g2x = k * (e3y * e1z - e3z * e1y), g2y = k * (e3z * e1x - e3x * e1z), g2z = k * (e3x * e1y - e3y * e1x);
            const float g3x = k * (e1y * e2z - e1z * e2y), g3y = k * (e1z * e2x - e1x * e2z), g3z = k * (e1x * e2y - e1y * e2x);
            if (!waited) {   // every row of this component must be stored before we add to it
              const unsigned int need = unsigned(hcur.expected);
              while (ld_acquire(p.done + hcur.comp) < need) __nanosleep(40);
              waited = true;
            }
            const size_t v0 = 3 * gid_x(tj[t][0]), v1 = 3 * gid_x(tj[t][1]), v2 = 3 * gid_x(tj[t][2]), v3 = 3 * gid_x(tj[t][3]);
            atomicAdd(grad + v0, -(g1x + g2x + g3x)); atomicAdd(grad + v0 + 1, -(g1y + g2y + g3y)); atomicAdd(grad + v0 + 2, -(g1z + g2z + g3z));
            atomicAdd(grad + v1, g1x); atomicAdd(grad + v1 + 1, g1y); atomicAdd(grad + v1 + 2, g1z);
            atomicAdd(grad + v2, g2x); atomicAdd(grad + v2 + 1, g2y); atomicAdd(grad + v2 + 2, g2z);
            atomicAdd(grad + v3, g3x); atomicAdd(grad + v3 + 1, g3y); atomicAdd(grad + v3 + 2, g3z);
          }
        } else if (AMIPS && amips_on && J > 0.f) {
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
          dea += double(tr / (3.f * j23) - 1.f);
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
            if (!waited) {
              const unsigned int need = unsigned(hcur.expected);
              while (ld_acquire(p.done + hcur.comp) < need) __nanosleep(40);
              waited = true;
            }
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
    }
    if (s == cs.x) TSB_STAMP(6);

    // ---- hand the staging buffers over ------------------------------------------------------------------
    if (s + 1 < cs.y) {      // (after the last segment the energy fold's own barrier is the only one needed)
      if (!GLOBAL) {
        if (li == 0 && eager2) {
          // segment 1 is already staged: no barrier
        } else {
          if (pre) {
            if (li == 1 && eager2) __syncthreads();     // half 0 is reused: every warp must have left segment 0
            store_staged(hn, li + 1);
          }
          __syncthreads();
          if (!pre) {
            stage_direct(hn, li + 1);
            __syncthreads();
          }
        }
      } else if (grad) {
        __syncthreads();     // keeps the named barrier's generations apart
      }
    }
    hcur = hn;
  }

  // ---- energies: lanes -> warp -> CTA partial; CTA 0 folds all partials in fixed order ---------------------
  TSB_STAMP(7);
  des = warp_sum(des);
  deb = warp_sum(deb);
  if (AMIPS) dea = warp_sum(dea);
  if (lane == 0) { red[3 * warp] = des; red[3 * warp + 1] = deb; red[3 * warp + 2] = dea; }
  __syncthreads();
  TSB_STAMP(8);
  if (tid == 0) {
    double a = 0.0, b = 0.0, c = 0.0;
    for (int w = 0; w < NW; ++w) { a += red[3 * w]; b += red[3 * w + 1]; c += red[3 * w + 2]; }
    a *= 0.5;
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
    if (lane == 0) {
      p.energy_out[0] = float(double(p.c1) * a + double(p.c2) * b + double(p.c3) * c3sum);
      p.energy_out[1] = float(a);
      p.energy_out[2] = float(b);
      if (p.energy4) p.energy_out[3] = float(c3sum);
    }
    for (int c = lane; c < p.n_components; c += 32) p.done[c] = 0u;   // every CTA has finished: safe to re-arm
  }
  TSB_STAMP(10);
#ifdef TSB_TRACE
  if (tid == 0 && p.trace) p.trace[blockIdx.x * 16 + 11] = gtime();
#endif
}

// GLOBAL mode pre-pass: u = x - X and x as float4 per vertex.
__global__ void prestage_kernel(const float *__restrict__ x, const float4 *__restrict__ X4, float4 *__restrict__ u4,
                                float4 *__restrict__ x4, int n) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    const float4 X = X4[v];
    const float a = x[3 * size_t(v)], b = x[3 * size_t(v) + 1], c = x[3 * size_t(v) + 2];
    u4[v] = make_float4(a - X.x, b - X.y, c - X.z, 0.f);
    x4[v] = make_float4(a, b, c, 0.f);
  }
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

template <int NW, int MINB, bool GLOBAL, bool AMIPS>
cudaError_t launch_variant(const KParams &p, const LaunchConfig &lc, cudaStream_t stream) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(unsigned(lc.grid));
  cfg.blockDim = dim3(NW * 32);
  cfg.dynamicSmemBytes = size_t(lc.smem_bytes);
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, energy_grad_kernel<NW, MINB, GLOBAL, AMIPS>, p);
}

template <int NW, int MINB, bool GLOBAL>
cudaError_t occupancy_variant(int smem_bytes, bool amips, int *ctas_per_sm) {
  // opt in to the device maximum once (the attribute is per function, not per handle: handles with different
  // staging sizes share the kernel)
  int dev = 0, optin = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e != cudaSuccess) return e;
  if (smem_bytes > optin) { *ctas_per_sm = 0; return cudaSuccess; }   // does not fit
  e = cudaFuncSetAttribute(energy_grad_kernel<NW, MINB, GLOBAL, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
  if (e == cudaSuccess && amips) e = cudaFuncSetAttribute(energy_grad_kernel<NW, MINB, GLOBAL, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
  if (e != cudaSuccess) { *ctas_per_sm = 0; cudaGetLastError(); return cudaSuccess; }
  int a = 0, b = 1 << 30;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, energy_grad_kernel<NW, MINB, GLOBAL, false>, NW * 32, size_t(smem_bytes));
  if (e == cudaSuccess && amips) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, energy_grad_kernel<NW, MINB, GLOBAL, true>, NW * 32, size_t(smem_bytes));
  *ctas_per_sm = a < b ? a : b;
  return e;
}

}  // namespace

int energy_ring_bytes(int slots, int cells_per_chunk, bool global) { return slots * cells_per_chunk * (global ? kCellGlobal : kCellStaged); }

int energy_smem_bytes(int nw, int ring_slots, int cells_per_chunk, int area_verts, bool global) {
  return smem_total(global ? 0 : area_verts * 32, nw, energy_ring_bytes(ring_slots, cells_per_chunk, global));
}

cudaError_t energy_occupancy(int nw, int smem_bytes, bool global, bool amips, int *ctas_per_sm) {
  if (nw == 16) return global ? occupancy_variant<16, 1, true>(smem_bytes, amips, ctas_per_sm) : occupancy_variant<16, 1, false>(smem_bytes, amips, ctas_per_sm);
  if (nw == 8) return global ? occupancy_variant<8, 2, true>(smem_bytes, amips, ctas_per_sm) : occupancy_variant<8, 2, false>(smem_bytes, amips, ctas_per_sm);
  return cudaErrorInvalidValue;
}

cudaError_t launch_energy_grad(const KParams &p, const LaunchConfig &lc, cudaStream_t stream) {
  if (lc.global) {
    prestage_kernel<<<grid_for(p.n, 256), 256, 0, stream>>>(p.x, p.X4, p.u4g, p.x4g, p.n);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if (lc.nw == 16) return lc.amips ? launch_variant<16, 1, true, true>(p, lc, stream) : launch_variant<16, 1, true, false>(p, lc, stream);
    if (lc.nw == 8) return lc.amips ? launch_variant<8, 2, true, true>(p, lc, stream) : launch_variant<8, 2, true, false>(p, lc, stream);
    return cudaErrorInvalidValue;
  }
  if (lc.nw == 16) return lc.amips ? launch_variant<16, 1, false, true>(p, lc, stream) : launch_variant<16, 1, false, false>(p, lc, stream);
  if (lc.nw == 8) return lc.amips ? launch_variant<8, 2, false, true>(p, lc, stream) : launch_variant<8, 2, false, false>(p, lc, stream);
  return cudaErrorInvalidValue;
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
