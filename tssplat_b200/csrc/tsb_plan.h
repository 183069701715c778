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
constexpr int kDetChunkRows = 256;                     // deterministic gather: vertex rows per chunk (= threads per CTA)

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
  int32_t deterministic = 0;    // also emit the vertex -> (tet slot, corner) lists of the deterministic gather (16 B per tet)
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
  std::vector<float> X4;            // STAGED: (X, Y, Z, 0) per staged vertex, component-major; GLOBAL: (X, Y, Z, bits
                                    // of the id of the component's reference vertex) by vertex id
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
  // Per component (per-sphere statistics).  Cuts run along the component-major cost stream and segs is CTA-major, so
  // the segments of a component are consecutive: component c owns segs[comp_seg[c], comp_seg[c + 1]).
  std::vector<int32_t> comp_seg;          // [n_components + 1]
  std::vector<int32_t> comp_first_vertex; // [n_components] lowest vertex id (components are numbered by it)
  std::vector<int32_t> comp_ntets;        // [n_components]
  std::vector<int32_t> comp_label;        // [n] component of every vertex, -1 = no tet references it (host only)
  // AMIPS only: rest inverses B = Dm^-1 of every streamed tet (in its streamed vertex order), one block of
  // 3 rows x (tets per cell) float4 per tet cell, and the first tet cell of every (segment, warp)
  std::vector<float> Bt;
  std::vector<int32_t> wtc0;        // also emitted for the deterministic gradient (it numbers the tet slots)
  // Deterministic gradient only.  Tet slot of a streamed tet: (wtc0[s, w] + tc) * (tets per cell) + lane * TPL + t.
  // Rows are the vertices of every component (components in order, vertices ascending); row r lists the entries
  // slot * 4 + corner of the non-padding tets whose streamed corner is det_vert[r], ascending.  Orphans have no row.
  std::vector<int32_t> det_rowptr;  // [rows + 1]
  std::vector<int32_t> det_vert;    // [rows] global vertex id
  std::vector<uint32_t> det_ent;    // [4 * nele] slot * 4 + corner
  std::vector<int32_t> det_comp_row;   // [n_components + 1] first row of every component
  std::vector<int32_t> det_chunk;   // [2 * chunks] (component, first row) of every run of <= kDetChunkRows rows
};

// The Newton-CG solver's view of the components (tsb_pcg_create): vert lists the non-orphan vertices grouped by
// component (components in order, vertices ascending), comp_off[c] is the first entry of component c, chunk holds
// (component, begin, end) for every run of <= kPcgChunkVerts entries of one component, components in order, and
// comp_chunk[c] is the first chunk of component c.
constexpr int kPcgChunkVerts = 256;
struct PcgLists {
  std::vector<int32_t> vert;        // [non-orphan vertices]
  std::vector<int32_t> comp_off;    // [n_components + 1]
  std::vector<int32_t> chunk;       // [3 * chunks]
  std::vector<int32_t> comp_chunk;  // [n_components + 1]
};
void build_pcg_lists(const std::vector<int32_t> &comp_label, int32_t n_components, PcgLists &out);

// Block pattern of the assembled Hessian (tsb_hessian_create): 3 x 3 block-CSR over all n vertex rows, the off-diagonal
// pattern of M plus the diagonal, columns ascending, no block between two components, orphan rows empty.  Every pair of
// vertices sharing a tet is a structural entry of M (build_rows keeps every column a tet stencil touches), which the
// builder checks while it fills tblk.
struct HessPattern {
  int64_t nnzb = 0;
  int64_t nnz = 0;                  // off-diagonal operator entries (= HostPlan::nnz of the same mesh)
  std::vector<int32_t> crow;        // [n + 1]
  std::vector<int32_t> col;         // [nnzb] global vertex ids
  std::vector<float> w;             // [nnzb] fp32 M_ij as the plan streams it; diagonal -sum_j M_ij (fp64, column order)
  std::vector<int32_t> tblk;        // [16 nele] block of corner pair (k, l) of tet t at 16 t + 4 k + l
  std::vector<int32_t> comp_label;  // [n] component of every vertex, -1 = orphan
};

// Returns 0 on success, TSB_E_* otherwise (message in err).
int build_hessian_pattern(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele, int32_t laplacian_scale,
                          HessPattern &out, std::string &err);

// The per-tet tables of the projected Hessian (tsb_pcg_enable_psd) and the assembled one (tsb_hessian_create).
struct TetTables {
  std::vector<int32_t> tets;        // [4 nele] the caller's vertex ids
  std::vector<float> B;             // [9][nele] rest inverse Dm^-1 (fp64, rounded), row-major entries
  std::vector<int32_t> inc_ptr;     // [n + 1]
  std::vector<int32_t> inc;         // [4 nele] 4 tet + corner, ascending within a vertex row
};

// Checks every tet in order: its vertices in [0, n), with comp_label (may be null) all four in one component, and a
// nonzero, finite rest volume.  Returns 0 on success, TSB_E_MESH for the first tet that fails (message in err).
int build_tet_tables(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele, const std::vector<int32_t> *comp_label,
                     TetTables &out, std::string &err);

// The affine coarse space of the per-component solve (tsb_pcg_enable_coarse), over the tables of build_tet_tables and the
// solver's PcgLists.  The tets are grouped by component (components in order, tet ids ascending in each) and cut into
// chunks of <= kCoarseTetChunk tets of one component: tchunk holds (component, begin, end) into tet, comp_tchunk[c] the
// first chunk of component c.  Y[3 e .. 3 e + 2] = X_v - mean_c X for entry e of PcgLists::vert (v its vertex, the mean
// over the component's vertices in fp64, the difference rounded to fp32); S[6 c ..] = sum_e Y_e Y_e^T of component c in
// fp64 from the fp32 Y, as 00 11 22 12 02 01.
constexpr int kCoarseTetChunk = 256;
struct CoarseTables {
  std::vector<int32_t> tet;          // [nele] tet ids grouped by component
  std::vector<int32_t> tets;         // [4 nele] their vertices
  std::vector<float> B;              // [9][nele] their Dm^-1, row-major entries
  std::vector<int32_t> tchunk;       // [3 * tet chunks]
  std::vector<int32_t> comp_tchunk;  // [n_components + 1]
  std::vector<float> Y;              // [3 rows]
  std::vector<double> S;             // [6 n_components]
};
// comp_label: the component of every vertex (every tet's vertices in one component, as build_tet_tables checks)
void build_coarse_tables(const float *rest_xyz, const TetTables &T, const std::vector<int32_t> &comp_label, const PcgLists &L,
                         CoarseTables &out);

// Multicolour symmetric Gauss-Seidel tables of the per-component solve (tsb_pcg_enable_sgs), over the block pattern crow /
// col of build_hessian_pattern and the solver's PcgLists.  Rows are numbered by their entry (position) in PcgLists::vert.
// Every component is coloured greedily on its own, vertices ascending, each vertex taking the smallest colour none of its
// earlier neighbours in the pattern holds; so the colours depend on neither the thread count nor the other components.
// lo[lo_ptr[e] .. lo_ptr[e + 1]) lists row e's blocks whose column has an earlier colour, hi the later ones, in column
// order, as (block index into the values array, position of the column in its component's vertex list).  sched holds the
// rows of every component grouped by colour (colours ascending, rows ascending in each); colour k of component c is
// sched[color_off[color_ptr[c] + k] .. color_off[color_ptr[c] + k + 1]).
struct SgsTables {
  int32_t n_colors = 0;             // the most colours any component uses
  std::vector<int32_t> color;       // [n] colour of every vertex, -1 = orphan
  std::vector<int32_t> lo_ptr, hi_ptr;   // [rows + 1]
  std::vector<int32_t> lo, hi;      // [2 * entries] (block, column position) pairs
  std::vector<int32_t> sched;       // [rows]
  std::vector<int32_t> color_ptr;   // [n_components + 1]
  std::vector<int32_t> color_off;   // [color_ptr[n_components]] (n_colors_c + 1 entries per component)
};
// nth: host threads (0: one per core, at most the plan builder's cap).  Returns 0 on success, TSB_E_* otherwise (message
// in err): a row of a component whose pattern has a column outside the component, or no diagonal block.
int build_sgs_tables(const std::vector<int32_t> &crow, const std::vector<int32_t> &col, const PcgLists &L, int nth,
                     SgsTables &out, std::string &err);

// Returns 0 on success, TSB_E_* otherwise (message in err).
int build_plan(const float *rest_xyz, const int32_t *tets, int32_t n, int32_t nele,
               const PlanConfig &cfg, HostPlan &plan, std::string &err);

}  // namespace tsb
