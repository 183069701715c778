// Host-side plan for the fused energy+gradient kernel (round-2 design: streamed operator rows).
//
// Replaces what the reference gets from libpgo at construction
// (tssplat_ext/tet_spheres/tet_spheres.cpp:140-203: pgo_create_tet_gradient_matrix and
// pgo_create_tet_biharmonic_gradient_matrix, uploaded as two COO matrices).  Like the reference we
// precompute the biharmonic operator M = G^T L^T L G (tet_spheres.cpp:148) once, in fp64, and round
// it to fp32 (tet_spheres.cpp:43-45) -- but we keep only its off-diagonal entries per vertex row
// (M has zero row sums, so (M u)_i = sum_{j != i} M_ij (u_j - u_i)) and lay them out as per-warp
// byte streams that TMA bulk copies pull through a shared-memory ring.  The barrier term needs, per
// tet, only its 4 vertex ids and 1/det(Dm) (det F = det(Ds) / det(Dm)); G itself is never stored.
//
// Work decomposition.  The mesh is cut into connected components (= tet-spheres; they share no
// vertices, geometry/tetmesh_geometry.py:305-331).  The cost stream of all components is cut into
// `grid` pieces, one per persistent CTA, with a fixed charge per piece so that cuts snap to component
// boundaries where they can; the piece of a component that lands in a CTA is a *segment*: a
// contiguous range of the component's vertex rows and of its tets.  A CTA stages the displacement
// u = x - X and the position x of the WHOLE component of each of its segments in shared memory
// (32 B per vertex), so every gather is a shared-memory read.  Inside a segment the rows are sorted
// by length and grouped into row blocks (RB) of 32 lanes, and the RBs plus the tet cells (64 tets
// STAGED, 32 GLOBAL) are dealt to the CTA's warps so that every warp has the same cost.
//
// Stream format v2 (per warp, segments back to back): a sequence of fixed-size CELLS, pulled through
// the warp's ring kCellsPerChunk cells per TMA copy; a cell is the unit, so no block depends on where
// a chunk or the ring ends.
//   STAGED (component-local vertex ids, stored as 16-bit BYTE OFFSETS from the start of the CTA's staging
//           area -- the plan knows which half-buffer a segment will use, so the kernel's gather address is
//           just smem_base + offset; row entries point at u, tet entries at x -- hence <= 1023 vertices
//           per double-buffered component and <= 2047 per "whole" component), cell = 768 B:
//     quad cell : u16 idx[32][4] | f32 w[32][4]     4 operator entries per lane
//     tet cell  : u16 idx[32][2][4] | f32 inv_det[32][2]   2 tets per lane (padding: 4 x vertex 0, inv_det 0)
//   GLOBAL (mesh-global 32-bit vertex ids), cell = 1024 B:
//     quad cell : u32 idx[32][4] | f32 w[32][4]
//     tet cell  : u32 idx[32][4] | f32 inv_det[32] | pad   1 tet per lane
// A row block (RB) is len4 consecutive quad cells.  Slot 0 of every lane's first quad is the RB header:
// idx = the lane's own row (so the gather returns u_i and the entry contributes exactly 0), and the
// weight's BIT PATTERN holds global row id (24 bits, 0xFFFFFF = idle lane) | len4 << 24 | log2(L) << 30
// (finite as a float because len4 <= 62, and it multiplies an exact 0).
// L = lanes per row (1, 2 or 4; the lanes of a row are adjacent and split its entries round-robin), chosen
// per block: when a segment's cells fit 90% of its CTA's rings (the latency regime of small problems) long
// rows are split until a block is at most half a ring, which shortens the per-warp serial chain; otherwise
// L = 1 unless a row needs more than 62 quad cells.  Padding slots: idx = a wildcard vertex, w = 0.
#pragma once
#include <cstdint>
#include <functional>
#include <memory>
#include <new>
#include <string>
#include <utility>
#include <vector>

namespace tsb {

constexpr int kCellStaged = 768, kCellGlobal = 1024;   // bytes per stream cell
constexpr int kMaxHalfVerts = 1023;                    // 64 * vh <= 65535 (16-bit byte offsets into the staging area)
constexpr int kMaxStagedVerts = 2047;                  // 32 * nv <= 65535
constexpr int kMaxWarps = 16;
constexpr int kCellsPerChunk = 6;                      // cells per TMA bulk copy = per ring slot (tsb_options_t.ring_slots)

// One segment (32 bytes).  comp indexes the per-component "rows done" counters; vbase >= 0 when the
// component's vertices are contiguous in the caller's numbering (then global id = vbase + local id),
// else -1 and vlist[x4off + local] holds the global id.
struct SegHdr {
  int32_t comp;
  int32_t vbase;
  int32_t nv;        // vertices of the component (all are staged)
  int32_t x4off;     // first entry of the component in X4 / vlist / pos16 (vertex order)
  int32_t expected;  // "rows stored" signals of this component = its number of segments (one per CTA piece)
  int32_t whole;     // 1: component needs the whole staging area (no double buffering around it)
  int32_t npos;      // staging positions of the component (>= nv: positions are bank-coloured, see pos16)
  int32_t p4off;     // first entry of the component in pos_gid (position order)
};
static_assert(sizeof(SegHdr) == 32, "SegHdr must be 32 bytes");

struct PlanConfig {
  int32_t nw = 16;              // warps per CTA
  int32_t grid = 132;           // persistent CTAs (used when grid_cb is empty; H100 SXM: 132 SMs)
  // Called once the component sizes are known, with the staging area the plan needs (vertices) and the mode
  // (true = GLOBAL; the callback may switch to it).  Sets grid and returns TSB_OK, or returns a TSB_E_* code
  // with a message in err.  Lets the caller size shared memory and query occupancy before the work is cut.
  std::function<int(int area_verts, bool &global_mode, int &grid, std::string &err)> grid_cb;
  int32_t vh_cap = kMaxHalfVerts;   // max vertices of a double-buffered ("half") component
  int32_t area_cap = kMaxStagedVerts;   // max vertices of any staged component (whole staging area)
  int32_t laplacian_scale = 0;
  int32_t force_global = 0;     // 1: skip staging, gather from global memory (testing / huge components)
  float tet_cost = 3.0f;        // cost of one tet relative to one operator entry (CTA-level cut)
  int32_t ring_cells = 2 * kCellsPerChunk;   // cells one warp's TMA ring holds (decides the latency / streaming regime)
  int32_t enable_amips = 0;     // also emit the per-tet rest inverses (AMIPS term; 48 B per tet)
};

// std::allocator whose construct() default-initialises: resize() of a byte vector does not zero-fill
// (the 306 MB stream of a 1024-sphere plan is first touched by the parallel copies that fill it)
template <class T>
struct NoInitAlloc : std::allocator<T> {
  template <class U> struct rebind { using other = NoInitAlloc<U>; };
  NoInitAlloc() = default;
  template <class U> NoInitAlloc(const NoInitAlloc<U> &) {}
  template <class U> void construct(U *p) noexcept { ::new (static_cast<void *>(p)) U; }
  template <class U, class... A> void construct(U *p, A &&...a) { ::new (static_cast<void *>(p)) U(std::forward<A>(a)...); }
};

struct HostPlan {
  int32_t n = 0, nele = 0, n_components = 0, n_boundary_faces = 0, laplacian_scale = 0;
  int32_t mode_global = 0;      // 0 = STAGED, 1 = GLOBAL
  int32_t nw = 0, grid = 0;
  int32_t vh = 0;               // half capacity actually needed (vertices)
  int32_t area_verts = 0;       // staging area actually needed (vertices)
  int32_t max_comp_verts = 0;
  int32_t contiguous = 1;       // every component has contiguous vertex ids (vlist unused)
  int64_t nnz = 0;              // off-diagonal operator entries
  int64_t nnz_padded = 0;       // entries stored (incl. row-block padding)
  int64_t n_rb = 0, n_tetcells = 0, n_cells = 0;
  int64_t gather_wavefronts[2] = {0, 0};   // STAGED row gathers: (wavefronts, ideal) per quarter-warp and slot
  int64_t tet_wavefronts[2] = {0, 0};

  std::vector<uint8_t, NoInitAlloc<uint8_t>> stream;   // all warp streams, 16-byte aligned (filled by parallel copies)
  std::vector<float> X4;            // 4 floats per staged vertex (X, Y, Z, 0), component-major
  std::vector<int32_t> vlist;       // global id per staged vertex (same order as X4)
  // Bank-aware placement: vertex k of a component is staged at position pos16[x4off + k] of its u / x
  // arrays; positions are chosen so that (position mod 8) -- the 16-byte shared-memory bank group of
  // the float4 -- is spread evenly over every operator row's columns, which lets the slot assignment
  // make the 8 gathers of a quarter-warp hit 8 different bank groups.
  std::vector<uint16_t> pos16;      // staging position per staged vertex (vertex order)
  std::vector<int32_t> pos_gid;     // global vertex id per staging position (position order, -1 = unused position)
  std::vector<SegHdr> segs;
  std::vector<int32_t> cta_seg;     // [2*grid] (first segment, one past last)
  std::vector<uint32_t> wdesc;      // [2*grid*nw] (stream offset / 16, stream bytes)
  std::vector<uint16_t> wseg;       // [2*nsegs*nw] (row blocks, tet cells) of each warp in each segment
  std::vector<int32_t> orphans;     // vertices no tet references (their gradient is zero)
  // AMIPS only: rest inverses B = Dm^-1 of every streamed tet (in its streamed vertex order), one block of
  // 3 rows x (tets per cell) float4 per tet cell, and the first tet cell of every (segment, warp)
  std::vector<float> Bt;
  std::vector<int32_t> wtc0;
};

// Returns 0 on success, TSB_E_* otherwise (message in err).
int build_plan(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele,
               const PlanConfig &cfg, HostPlan &plan, std::string &err);

}  // namespace tsb
