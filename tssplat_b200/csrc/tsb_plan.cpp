// Host plan builder: validation, face adjacency, connected components, the fp64 biharmonic operator
// rows (M = G^T L^T L G, off-diagonal part), 1/det(Dm) per tet, cost-balanced segmentation over the
// persistent CTAs and their warps, and the per-warp TMA byte streams.  See tsb_plan.h.
#include "tsb_plan.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <numeric>
#include <thread>

#include "../../include/tssplat_b200.h"

namespace tsb {
namespace {

struct FaceKey {
  uint32_t a, b, c, owner;  // sorted vertex triple; owner = 4*tet + local face
  bool operator<(const FaceKey &o) const {
    if (a != o.a) return a < o.a;
    if (b != o.b) return b < o.b;
    return c < o.c;
  }
  bool same(const FaceKey &o) const { return a == o.a && b == o.b && c == o.c; }
};

// Face k of a tet is the face opposite to local vertex k.
const int kFace[4][3] = {{1, 2, 3}, {0, 3, 2}, {0, 1, 3}, {0, 2, 1}};

struct UnionFind {
  std::vector<int32_t> p;
  explicit UnionFind(int n) : p(n) { std::iota(p.begin(), p.end(), 0); }
  int find(int x) {
    while (p[x] != x) { p[x] = p[p[x]]; x = p[x]; }
    return x;
  }
  void unite(int a, int b) {
    a = find(a); b = find(b);
    if (a != b) p[std::max(a, b)] = std::min(a, b);
  }
};

// B = Dm^-1 (row-major) and det(Dm) of the tet with vertices v[0..3] in this order (Dm column k = X_{k+1} - X_0).
// Returns false for a degenerate tet.
bool rest_inverse(const float *rest, const int32_t *v, double *o, double *det) {
  double m[9];
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k) m[3 * r + k] = double(rest[3 * size_t(v[k + 1]) + r]) - double(rest[3 * size_t(v[0]) + r]);
  const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
  const double d = m[0] * c00 + m[1] * c01 + m[2] * c02;
  if (d == 0.0 || !std::isfinite(d)) return false;
  const double id = 1.0 / d;
  o[0] = c00 * id; o[1] = (m[2] * m[7] - m[1] * m[8]) * id; o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
  o[3] = c01 * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  o[6] = c02 * id; o[7] = (m[1] * m[6] - m[0] * m[7]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
  *det = d;
  return true;
}

// One connected component: its vertices (sorted global ids), tets, and operator rows.
struct Comp {
  std::vector<int32_t> verts;   // sorted global ids; local id = position
  std::vector<int32_t> tets;    // global tet ids, ascending
  std::vector<int32_t> rptr;    // [nv+1]
  std::vector<int32_t> col;     // local column ids (sorted inside a row), off-diagonal only
  std::vector<float> val;
  std::vector<int32_t> pos;     // staging position of each local vertex (bank-coloured); identity in GLOBAL mode
  int32_t npos = 0;             // positions used (8 * largest colour class)
  int32_t first_of_color[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // a vertex with each (position mod 8): wildcard padding targets
  int32_t contiguous = 1;
};

struct Mesh {
  const float *rest;
  const int32_t *tets;
  int32_t n, nele;
  std::vector<int32_t> nbr;       // [4*nele] neighbour tet across face k, -1 = boundary
  std::vector<int32_t> local_of;  // [n] local id of a vertex inside its component
  int32_t lap_scale;
};

// Face adjacency of one component (faces never cross components): sort the 4 face keys of its tets and pair
// equal neighbours.  Returns the number of boundary faces, or -1 for a face shared by more than two tets.
int64_t build_adjacency(Mesh &M, const Comp &C) {
  std::vector<FaceKey> fk(C.tets.size() * 4);
  for (size_t i = 0; i < C.tets.size(); ++i) {
    const int32_t t = C.tets[i];
    const int32_t *v = M.tets + 4 * size_t(t);
    for (int k = 0; k < 4; ++k) {
      uint32_t f[3] = {uint32_t(v[kFace[k][0]]), uint32_t(v[kFace[k][1]]), uint32_t(v[kFace[k][2]])};
      if (f[0] > f[1]) std::swap(f[0], f[1]);
      if (f[1] > f[2]) std::swap(f[1], f[2]);
      if (f[0] > f[1]) std::swap(f[0], f[1]);
      fk[4 * i + k] = FaceKey{f[0], f[1], f[2], uint32_t(4 * t + k)};
    }
  }
  std::sort(fk.begin(), fk.end());
  int64_t boundary = 0;
  const size_t nf = fk.size();
  for (size_t i = 0; i < nf;) {
    size_t j = i + 1;
    while (j < nf && fk[j].same(fk[i])) ++j;
    if (j - i > 2) return -1;
    if (j - i == 2) {
      const uint32_t o0 = fk[i].owner, o1 = fk[i + 1].owner;
      M.nbr[o0] = int32_t(o1 >> 2);
      M.nbr[o1] = int32_t(o0 >> 2);
    } else {
      ++boundary;
    }
    i = j;
  }
  return boundary;
}

// Rows of M = G^T L^T L G for one component, in fp64, off-diagonal entries rounded to fp32.
//   F_t = sum_v x_v (x) a_{t,v}  (a = rest gradients of the hat functions: rows of Dm^-1, geometry/mesh_utils.py:38-69)
//   (L F)_t = w_t (deg_t F_t - sum_{s ~ t} F_s) = sum_v x_v (x) W_{t,v},   W_{t,v} = w_t (deg_t a_{t,v} - sum_s a_{s,v})
//   M_ij = sum_t W_{t,i} . W_{t,j}          (per coordinate; the reference's matrix is M (x) I_3)
// L is the face-adjacency graph Laplacian of the tets (THE libpgo assumption, oracle/tet_energy_oracle.py:
// tet_laplacian), w_t = 1 (unscaled, what the reference requests) or 1/deg_t (laplacian_scale = 1).
void build_rows(const Mesh &M, Comp &C) {
  const int nv = int(C.verts.size()), nt = int(C.tets.size());
  // hat gradients of every tet of the component (fp64)
  std::vector<double> A(size_t(nt) * 12);
  for (int tl = 0; tl < nt; ++tl) {
    double B[9], det;
    rest_inverse(M.rest, M.tets + 4 * size_t(C.tets[tl]), B, &det);   // validated earlier
    double *a = &A[size_t(tl) * 12];
    for (int c = 0; c < 3; ++c) {
      a[3 + c] = B[c]; a[6 + c] = B[3 + c]; a[9 + c] = B[6 + c];
      a[c] = -(B[c] + B[3 + c] + B[6 + c]);
    }
  }
  // local tet lookup through a sorted search (component tets are ascending)
  auto tl_find = [&](int32_t t) { return int(std::lower_bound(C.tets.begin(), C.tets.end(), t) - C.tets.begin()); };

  // per-tet stencils: up to 8 (vertex, W) pairs
  struct Ent { int32_t v; double w[3]; };
  std::vector<Ent> st(size_t(nt) * 8);
  std::vector<uint8_t> cnt(nt, 0);
  std::vector<int32_t> inc_ptr(size_t(nv) + 1, 0);
  for (int tl = 0; tl < nt; ++tl) {
    const int32_t t = C.tets[tl];
    Ent *e = &st[size_t(tl) * 8];
    int ne = 0;
    int deg = 0;
    for (int k = 0; k < 4; ++k) deg += M.nbr[4 * size_t(t) + k] >= 0;
    const double wt = M.lap_scale ? (deg > 0 ? 1.0 / deg : 0.0) : 1.0;
    auto add = [&](int32_t vloc, const double *a, double coef) {
      for (int i = 0; i < ne; ++i)
        if (e[i].v == vloc) { for (int c = 0; c < 3; ++c) e[i].w[c] += coef * a[c]; return; }
      e[ne].v = vloc;
      for (int c = 0; c < 3; ++c) e[ne].w[c] = coef * a[c];
      ++ne;
    };
    const int32_t *v = M.tets + 4 * size_t(t);
    for (int k = 0; k < 4; ++k) add(M.local_of[v[k]], &A[size_t(tl) * 12 + 3 * k], wt * deg);
    for (int f = 0; f < 4; ++f) {
      const int32_t s = M.nbr[4 * size_t(t) + f];
      if (s < 0) continue;
      const int sl = tl_find(s);
      const int32_t *vs = M.tets + 4 * size_t(s);
      for (int k = 0; k < 4; ++k) add(M.local_of[vs[k]], &A[size_t(sl) * 12 + 3 * k], -wt);
    }
    cnt[tl] = uint8_t(ne);
    for (int i = 0; i < ne; ++i) ++inc_ptr[e[i].v + 1];
  }
  for (int i = 0; i < nv; ++i) inc_ptr[i + 1] += inc_ptr[i];
  std::vector<int32_t> inc(static_cast<size_t>(inc_ptr[nv]), 0);   // (tl * 8 + slot)
  {
    std::vector<int32_t> cur(inc_ptr.begin(), inc_ptr.end() - 1);
    for (int tl = 0; tl < nt; ++tl)
      for (int i = 0; i < cnt[tl]; ++i) inc[cur[st[size_t(tl) * 8 + i].v]++] = tl * 8 + i;
  }
  // rows
  C.rptr.assign(size_t(nv) + 1, 0);
  C.col.clear(); C.val.clear();
  C.col.reserve(size_t(nv) * 40); C.val.reserve(size_t(nv) * 40);
  std::vector<double> acc(nv, 0.0);
  std::vector<uint8_t> seen(nv, 0);
  std::vector<int32_t> touched;
  for (int i = 0; i < nv; ++i) {
    touched.clear();
    for (int32_t p = inc_ptr[i]; p < inc_ptr[i + 1]; ++p) {
      const int tl = inc[p] >> 3, si = inc[p] & 7;
      const Ent *e = &st[size_t(tl) * 8];
      const double *wi = e[si].w;
      for (int j = 0; j < cnt[tl]; ++j) {
        const int32_t vj = e[j].v;
        if (vj == i) continue;
        if (!seen[vj]) { seen[vj] = 1; touched.push_back(vj); }
        acc[vj] += wi[0] * e[j].w[0] + wi[1] * e[j].w[1] + wi[2] * e[j].w[2];
      }
    }
    std::sort(touched.begin(), touched.end());
    for (int32_t vj : touched) {
      C.col.push_back(vj);
      C.val.push_back(float(acc[vj]));      // fp64 -> fp32 like the reference's operators (tet_spheres.cpp:43-45)
      acc[vj] = 0.0; seen[vj] = 0;
    }
    C.rptr[i + 1] = int32_t(C.col.size());
  }
}

// Bank-aware staging positions (see HostPlan::pos16).  Greedy balanced 8-colouring of the operator's
// sparsity graph: a vertex takes the colour that is rarest among the columns of the rows it appears in
// (the pattern is symmetric, so those rows are its own columns); position = 8 * (rank in colour) + colour.
void place_vertices(Comp &C, bool identity) {
  const int nv = int(C.verts.size());
  C.pos.resize(nv);
  if (identity || nv < 64) {
    for (int v = 0; v < nv; ++v) C.pos[v] = v;
    C.npos = nv;
    for (int c = 0; c < 8; ++c) C.first_of_color[c] = c < nv ? c : 0;
    return;
  }
  std::vector<int32_t> cnt(size_t(nv) * 8, 0);
  std::vector<int32_t> order(nv), color(nv, -1);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return C.rptr[a + 1] - C.rptr[a] > C.rptr[b + 1] - C.rptr[b]; });
  int glob[8] = {0};
  for (int sweep = 0; sweep < 2; ++sweep) {
    for (int v : order) {
      const int32_t *nb = &C.col[size_t(C.rptr[v])];
      const int deg = C.rptr[v + 1] - C.rptr[v];
      if (color[v] >= 0) {
        for (int k = 0; k < deg; ++k) --cnt[size_t(nb[k]) * 8 + color[v]];
        --glob[color[v]];
      }
      int64_t cost[8] = {0};
      for (int k = 0; k < deg; ++k)
        for (int c = 0; c < 8; ++c) cost[c] += cnt[size_t(nb[k]) * 8 + c];
      int best = 0;
      for (int c = 1; c < 8; ++c)
        if (cost[c] * 1024 + glob[c] < cost[best] * 1024 + glob[best]) best = c;
      color[v] = best;
      for (int k = 0; k < deg; ++k) ++cnt[size_t(nb[k]) * 8 + best];
      ++glob[best];
    }
  }
  int rank[8] = {0};
  for (int c = 0; c < 8; ++c) C.first_of_color[c] = -1;
  for (int v = 0; v < nv; ++v) {
    const int c = color[v];
    C.pos[v] = 8 * rank[c]++ + c;
    if (C.first_of_color[c] < 0) C.first_of_color[c] = v;
  }
  int mx = 0;
  for (int c = 0; c < 8; ++c) { mx = std::max(mx, rank[c]); if (C.first_of_color[c] < 0) C.first_of_color[c] = 0; }
  C.npos = 8 * mx;
}

template <class T>
void put(std::vector<uint8_t> &b, size_t off, T v) { std::memcpy(b.data() + off, &v, sizeof(T)); }

struct RowRef { int32_t row; int32_t len; };

// quad cells an RB of these rows needs when each row is split over L lanes (slot 0 of a lane = header)
inline int rb_len4(const RowRef *rows, int nrows, int L) {
  int len4 = 1;
  for (int i = 0; i < nrows; ++i) {
    const int per_lane = (rows[i].len + L - 1) / L;       // lane 0 of the row holds the most
    len4 = std::max(len4, (per_lane + 1 + 3) / 4);
  }
  return len4;
}

// Shared-memory bank model of the kernel's 128-bit gathers: a quarter-warp (8 adjacent lanes) is served
// in one wavefront when its 8 float4 addresses fall into 8 different 16-byte bank groups, i.e. when the
// vertex ids differ mod 8 (all lanes add the same base).  Within a row the order of the entries is free
// and padding slots may point at ANY vertex (their weight is 0), so for every slot column we match the 8
// lanes of a quarter to 8 distinct residues.  Returns the slot layout: slot_col[lane][slot] (local vertex
// id, -1 = wildcard padding that still needs a residue) and slot_ent[lane][slot] (entry index or -1).
struct LaneSlots {
  std::vector<int32_t> col;   // [32 * nslots] local column id per (lane, slot)
  std::vector<int32_t> ent;   // [32 * nslots] entry index inside the lane's row, -1 = padding
};

void assign_slots(const Comp &C, const RowRef *rows, int nrows, int L, int len4, LaneSlots &out) {
  const int nslots = 4 * len4, NC = nslots - 1;       // colours = slots 1..nslots-1 (slot 0 is the header)
  out.col.assign(size_t(32) * nslots, 0);
  out.ent.assign(size_t(32) * nslots, -1);
  int own[32];
  for (int l = 0; l < 32; ++l) {
    const int ri = l / L;
    own[l] = ri < nrows ? rows[ri].row : 0;
    out.col[size_t(l) * nslots] = own[l];             // slot 0 = header (own row)
  }
  // Per quarter-warp: proper edge colouring of the bipartite multigraph lanes x residues (one edge per
  // operator entry, colour = slot).  Konig: possible with NC colours whenever no residue has more than NC
  // entries among the quarter's 8 lanes; the few excess edges go to any free slot of their lane.
  std::vector<int32_t> lane_ent(size_t(8) * NC), lane_res(size_t(8) * NC), res_lane(size_t(8) * NC);
  std::vector<int32_t> overflow;
  for (int q = 0; q < 4; ++q) {
    std::fill(lane_ent.begin(), lane_ent.end(), -1);
    std::fill(lane_res.begin(), lane_res.end(), -1);
    std::fill(res_lane.begin(), res_lane.end(), -1);
    int lane_deg[8] = {0}, res_deg[8] = {0};
    auto L_ = [&](int i, int c) -> int32_t & { return lane_res[size_t(i) * NC + c]; };   // residue of lane i's edge coloured c
    auto E_ = [&](int i, int c) -> int32_t & { return lane_ent[size_t(i) * NC + c]; };   // its entry index
    auto R_ = [&](int r, int c) -> int32_t & { return res_lane[size_t(r) * NC + c]; };   // lane of residue r's edge coloured c
    overflow.clear();
    for (int i = 0; i < 8; ++i) {
      const int l = 8 * q + i, ri = l / L, sub = l % L;
      if (ri >= nrows) continue;
      const int row = rows[ri].row, len = rows[ri].len;
      const int32_t *col = &C.col[size_t(C.rptr[row])];
      for (int e = sub; e < len; e += L) {
        const int r = C.pos[col[e]] & 7;
        if (res_deg[r] >= NC) { overflow.push_back(i * 65536 + e); continue; }   // residue saturated: unavoidable conflict
        int a = 0, b = 0;
        while (L_(i, a) >= 0) ++a;                     // free at the lane (lane degree <= NC by construction)
        while (R_(r, b) >= 0) ++b;                     // free at the residue
        if (R_(r, a) >= 0) {                           // a is taken at r: flip the a/b alternating path that starts at r
          int rr = r, ca = a, cb = b;
          // collect the path edges (lane, colour) then swap
          int path_lane[64], path_col[64], np = 0;
          int cur_r = rr;
          bool at_res = true;
          int cur_l = -1;
          while (np < 64) {
            if (at_res) {
              const int ln = R_(cur_r, ca);
              if (ln < 0) break;
              path_lane[np] = ln; path_col[np] = ca; ++np;
              cur_l = ln; at_res = false;
            } else {
              const int rn = L_(cur_l, cb);
              if (rn < 0) break;
              path_lane[np] = cur_l; path_col[np] = cb; ++np;
              cur_r = rn; at_res = true;
            }
          }
          // remove all path edges, then re-insert with swapped colours
          int pe[64], pr[64];
          for (int k = 0; k < np; ++k) {
            const int ln = path_lane[k], c = path_col[k];
            pe[k] = E_(ln, c); pr[k] = L_(ln, c);
            R_(pr[k], c) = -1; L_(ln, c) = -1; E_(ln, c) = -1;
          }
          for (int k = 0; k < np; ++k) {
            const int ln = path_lane[k], c = path_col[k] == ca ? cb : ca;
            L_(ln, c) = pr[k]; E_(ln, c) = pe[k]; R_(pr[k], c) = ln;
          }
        }
        L_(i, a) = r; E_(i, a) = e; R_(r, a) = i;
        ++lane_deg[i]; ++res_deg[r];
      }
    }
    for (int32_t oe : overflow) {                       // excess edges: any free slot of the lane
      const int i = oe >> 16, e = oe & 0xFFFF;
      int a = 0;
      while (L_(i, a) >= 0) ++a;
      L_(i, a) = 8;                                     // marks "placed, conflicts allowed"
      E_(i, a) = e;
    }
    for (int c = 0; c < NC; ++c) {
      uint32_t used = 0;
      for (int i = 0; i < 8; ++i) if (L_(i, c) >= 0 && L_(i, c) < 8) used |= 1u << L_(i, c);
      for (int i = 0; i < 8; ++i) {
        const int l = 8 * q + i;
        int32_t col_out;
        if (E_(i, c) >= 0) {
          col_out = C.col[size_t(C.rptr[own[l]]) + E_(i, c)];
        } else {                                        // padding: any vertex with a residue nobody uses in this slot
          int r = -1;
          for (int k = 0; k < 8; ++k) if (!((used >> k) & 1u)) { r = k; break; }
          if (r >= 0) { used |= 1u << r; col_out = C.first_of_color[r]; } else col_out = own[l];
        }
        out.col[size_t(l) * nslots + 1 + c] = col_out;
        out.ent[size_t(l) * nslots + 1 + c] = E_(i, c);
      }
    }
  }
}

// Appends one row block (len4 quad cells).  STAGED: IDX = uint16_t byte offsets into the staging area;
// GLOBAL: IDX = uint32_t global ids (gid maps local -> global).  Returns len4.
template <class IDX>
int emit_rb(std::vector<uint8_t> &s, const Comp &C, const RowRef *rows, int nrows, int L, const int32_t *gid, int ubase_bytes,
            LaneSlots &scratch, int64_t *conflict_stat) {
  constexpr bool kGlobal = sizeof(IDX) == 4;
  constexpr size_t CELL = kGlobal ? kCellGlobal : kCellStaged, WOFF = 128 * sizeof(IDX);
  const int len4 = rb_len4(rows, nrows, L);
  const int nslots = 4 * len4;
  int llog = 0;
  while ((1 << llog) < L) ++llog;
  auto stored = [&](int32_t local) -> IDX { return kGlobal ? IDX(gid[local]) : IDX(ubase_bytes + C.pos[local] * 16); };
  // Lane order inside the block is free: deal the rows to the four quarter-warps so that the header
  // gathers (slot 0: every lane reads its own row) also hit distinct bank groups.
  RowRef arranged[32];
  if (L == 1 && !kGlobal) {
    int fill[4] = {0, 0, 0, 0};
    uint32_t qused[4] = {0, 0, 0, 0};
    RowRef tmp[4][8];
    std::vector<int> later;
    for (int i = 0; i < nrows; ++i) {
      const int r = C.pos[rows[i].row] & 7;
      int best = -1;
      for (int q = 0; q < 4; ++q)
        if (fill[q] < 8 && !((qused[q] >> r) & 1u) && (best < 0 || fill[q] < fill[best])) best = q;
      if (best < 0) { later.push_back(i); continue; }
      tmp[best][fill[best]++] = rows[i];
      qused[best] |= 1u << r;
    }
    for (int i : later) {
      int best = 0;
      for (int q = 1; q < 4; ++q) if (fill[q] < fill[best]) best = q;
      tmp[best][fill[best]++] = rows[i];
    }
    // lanes of a quarter must be contiguous and idle lanes last: quarters are filled 0..3 in order of size
    int order4[4] = {0, 1, 2, 3};
    std::sort(order4, order4 + 4, [&](int a, int b) { return fill[a] > fill[b]; });
    // idle lanes may only trail the active ones (rows[ri] with ri >= nrows is idle): compact quarter by quarter,
    // keeping every full quarter intact
    int n = 0;
    for (int k = 0; k < 4; ++k)
      for (int i = 0; i < fill[order4[k]]; ++i) arranged[n++] = tmp[order4[k]][i];
    rows = arranged;
  }
  assign_slots(C, rows, nrows, L, len4, scratch);
  size_t o = s.size();
  s.resize(o + size_t(len4) * CELL, 0);
  for (int l = 0; l < 32; ++l) {
    const int ri = l / L;
    const bool active = ri < nrows;
    const int r = active ? rows[ri].row : 0;
    const float *val = active ? &C.val[size_t(C.rptr[r])] : nullptr;
    for (int slot = 0; slot < nslots; ++slot) {
      const IDX id = stored(scratch.col[size_t(l) * nslots + slot]);
      uint32_t wbits = 0;
      if (slot == 0) {
        // header: global row id (24 bits, 0xFFFFFF = idle lane) | len4 << 24 | log2(L) << 30.  Read as a float it
        // is finite (len4 <= 62 keeps the exponent below 0xFF) and it multiplies a difference that is exactly 0.
        const uint32_t rid = active ? uint32_t(kGlobal ? gid[r] : C.verts[r]) : 0xFFFFFFu;
        wbits = rid | (uint32_t(len4) << 24) | (uint32_t(llog) << 30);
      } else {
        const int e = scratch.ent[size_t(l) * nslots + slot];
        if (e >= 0) std::memcpy(&wbits, &val[e], 4);
      }
      const size_t cell = o + size_t(slot / 4) * CELL;
      put<IDX>(s, cell + (size_t(l) * 4 + (slot & 3)) * sizeof(IDX), id);
      put<uint32_t>(s, cell + WOFF + (size_t(l) * 4 + (slot & 3)) * 4, wbits);
    }
  }
  if (conflict_stat) {      // wavefronts of the gathers: ideal = 1 per (quarter, slot)
    for (int q = 0; q < 4; ++q)
      for (int slot = 0; slot < nslots; ++slot) {
        int cnt[8] = {0};
        int32_t first[8];
        for (int k = 0; k < 8; ++k) first[k] = -1;
        int worst = 1;
        for (int i = 0; i < 8; ++i) {
          const int32_t c = C.pos[scratch.col[size_t(8 * q + i) * nslots + slot]];
          const int r = c & 7;
          if (first[r] == c) continue;              // same address: broadcast, no extra wavefront
          if (first[r] < 0) first[r] = c;
          ++cnt[r];
          worst = std::max(worst, cnt[r]);
        }
        conflict_stat[0] += worst;
        conflict_stat[1] += 1;
      }
  }
  return len4;
}

// Appends one tet cell: STAGED 64 tets (2 per lane), GLOBAL 32 tets.
template <class IDX>
void emit_tc(std::vector<uint8_t> &s, const Mesh &M, const Comp &C, int t0, int nt, int xbase_bytes, int64_t *stat, std::vector<float> *Bout) {
  constexpr bool kGlobal = sizeof(IDX) == 4;
  constexpr size_t CELL = kGlobal ? kCellGlobal : kCellStaged;
  constexpr int TPL = kGlobal ? 1 : 2;
  constexpr size_t DOFF = 32 * TPL * 4 * sizeof(IDX);
  size_t o = s.size();
  s.resize(o + CELL, 0);
  if (!kGlobal)   // padding tets: four times the component's vertex 0 (det 0) with 1/det(Dm) = 0
    for (int i = 0; i < 32 * TPL * 4; ++i) put<IDX>(s, o + size_t(i) * sizeof(IDX), IDX(xbase_bytes + C.pos[0] * 16));
  // The barrier is invariant under any relabelling of a tet's vertices as long as 1/det(Dm) is taken for
  // the same order, so each tet's vertex order is chosen to give the 8 lanes of a quarter-warp distinct
  // bank groups in each of its 4 gathers (greedy over the 24 permutations).
  static const uint8_t kPerm[24][4] = {{0,1,2,3},{0,1,3,2},{0,2,1,3},{0,2,3,1},{0,3,1,2},{0,3,2,1},{1,0,2,3},{1,0,3,2},{1,2,0,3},{1,2,3,0},{1,3,0,2},{1,3,2,0},
                                       {2,0,1,3},{2,0,3,1},{2,1,0,3},{2,1,3,0},{2,3,0,1},{2,3,1,0},{3,0,1,2},{3,0,2,1},{3,1,0,2},{3,1,2,0},{3,2,0,1},{3,2,1,0}};
  size_t bo = 0;
  if (Bout) { bo = Bout->size(); Bout->resize(bo + size_t(3) * 32 * TPL * 4, 0.f); }   // [row][lane*TPL + k] float4
  // choose the vertex order of every tet: min-conflicts over each group of 8 lanes x one tet slot
  std::vector<uint8_t> perm_of(size_t(nt), 0);
  if (!kGlobal) {
    const int ngroups = 4 * TPL;                      // (quarter, slot)
    for (int gq = 0; gq < ngroups; ++gq) {
      const int q = gq / TPL, k = gq % TPL;
      int members[8], nm = 0, pos4[8][4];
      for (int i8 = 0; i8 < 8; ++i8) {
        const int i = (8 * q + i8) * TPL + k;         // tet index inside the cell: lane * TPL + slot
        if (i >= nt) continue;
        const int32_t *v0 = M.tets + 4 * size_t(C.tets[size_t(t0) + i]);
        for (int c = 0; c < 4; ++c) pos4[nm][c] = C.pos[M.local_of[v0[c]]];
        members[nm++] = i;
      }
      // cost of placing vertex position p in gather c: lanes already reading the same bank group at a
      // DIFFERENT address (same address = broadcast, free)
      int cur[8];
      auto conflicts = [&](int m, int pi) {
        int hits = 0;
        for (int c = 0; c < 4; ++c) {
          const int p = pos4[m][kPerm[pi][c]];
          for (int o = 0; o < nm; ++o) {
            if (o == m || cur[o] < 0) continue;
            const int po = pos4[o][kPerm[cur[o]][c]];
            hits += ((po & 7) == (p & 7)) && po != p;
          }
        }
        return hits;
      };
      for (int m = 0; m < nm; ++m) cur[m] = -1;
      for (int m = 0; m < nm; ++m) {                  // greedy start
        int best = 0, best_hits = 1 << 30;
        for (int pi = 0; pi < 24; ++pi) {
          const int hits = conflicts(m, pi);
          if (hits < best_hits) { best_hits = hits; best = pi; if (!hits) break; }
        }
        cur[m] = best;
      }
      for (int sweep = 0; sweep < 4; ++sweep) {       // local repair
        bool changed = false;
        for (int m = 0; m < nm; ++m) {
          int best = cur[m], best_hits = conflicts(m, cur[m]);
          if (!best_hits) continue;
          for (int pi = 0; pi < 24; ++pi) {
            const int hits = conflicts(m, pi);
            if (hits < best_hits) { best_hits = hits; best = pi; }
          }
          if (best != cur[m]) { cur[m] = best; changed = true; }
        }
        if (!changed) break;
      }
      if (stat)
        for (int c = 0; c < 4; ++c) {                  // wavefronts of this gather = max distinct addresses per bank group
          int worst = 1;
          for (int r = 0; r < 8; ++r) {
            int distinct = 0, seen[8];
            for (int m = 0; m < nm; ++m) {
              const int p = pos4[m][kPerm[cur[m]][c]];
              if ((p & 7) != r) continue;
              bool dup = false;
              for (int d = 0; d < distinct; ++d) dup |= seen[d] == p;
              if (!dup) seen[distinct++] = p;
            }
            worst = std::max(worst, distinct);
          }
          stat[0] += worst; stat[1] += 1;
        }
      for (int m = 0; m < nm; ++m) perm_of[members[m]] = uint8_t(cur[m]);
    }
  }
  for (int i = 0; i < nt; ++i) {
    const int l = i / TPL, k = i % TPL;          // lane, tet slot inside the lane
    const int32_t t = C.tets[size_t(t0) + i];
    const int32_t *v0 = M.tets + 4 * size_t(t);
    int32_t v[4];
    for (int c = 0; c < 4; ++c) v[c] = v0[kPerm[perm_of[i]][c]];
    double B[9], det;
    rest_inverse(M.rest, v, B, &det);
    for (int c = 0; c < 4; ++c)
      put<IDX>(s, o + ((size_t(l) * TPL + k) * 4 + c) * sizeof(IDX), kGlobal ? IDX(v[c]) : IDX(xbase_bytes + C.pos[M.local_of[v[c]]] * 16));
    put<float>(s, o + DOFF + (size_t(l) * TPL + k) * 4, float(1.0 / det));
    if (Bout)
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) (*Bout)[bo + (size_t(r) * 32 * TPL + size_t(l) * TPL + k) * 4 + c] = float(B[3 * r + c]);
  }
}

constexpr int kMaxHostThreads = 32;
constexpr double kRowCost = 2.0;        // cost of one vertex row (header, store) in operator entries (CTA-level cut)
constexpr float kTetCellCost = 1.3f;    // cost of one tet cell relative to one quad cell (warp-level deal)
constexpr float kSegOverhead = 0.60f;   // fixed cost of every (CTA, component) segment, as a fraction of the mean CTA cost
constexpr int kMaxLanesPerRow = 4;      // rows may be split over up to this many adjacent lanes (latency regime only)
constexpr int kRbCapDiv = 2;            // latency regime: a row block is at most ring_cells / kRbCapDiv quad cells

// Runs fn(begin, end) over [0, count) in chunks of `grain` items, handed out in order to up to `nth` host threads
// (the calling one included) as they become free.  The items of every phase are independent, so the plan does not
// depend on how they are split.
template <class F>
void parallel_for(size_t count, size_t grain, int nth, F fn) {
  const size_t chunks = (count + grain - 1) / grain;
  std::atomic<size_t> next{0};
  auto work = [&] {
    for (size_t c = next++; c < chunks; c = next++) fn(c * grain, std::min(count, (c + 1) * grain));
  };
  std::vector<std::thread> th;
  for (size_t k = 1; k < std::min(chunks, size_t(nth)); ++k) th.emplace_back(work);
  work();
  for (auto &t : th) t.join();
}

// What is wrong with the tet with vertices v[0..3], or nullptr.  Checked in this order: vertex index out of
// range, repeated vertex, zero rest volume.
const char *tet_problem(const float *rest, const int32_t *v, int32_t n) {
  for (int k = 0; k < 4; ++k)
    if (v[k] < 0 || v[k] >= n) return "has a vertex index out of range";
  if (v[0] == v[1] || v[0] == v[2] || v[0] == v[3] || v[1] == v[2] || v[1] == v[3] || v[2] == v[3]) return "repeats a vertex";
  double B[9], det;
  if (!rest_inverse(rest, v, B, &det) || !std::isfinite(float(1.0 / det))) return "has zero rest volume";
  return nullptr;
}

// Reports the lowest offending tet, like a serial scan would.
int validate(const float *rest, const int32_t *tets, int32_t n, int32_t nele, int nth, std::string &err) {
  std::atomic<int> bad_tet{nele};
  parallel_for(size_t(nele), 8192, nth, [&](size_t b, size_t e) {
    for (size_t t = b; t < e; ++t)
      if (tet_problem(rest, tets + 4 * t, n)) {
        int cur = bad_tet.load();
        while (int(t) < cur && !bad_tet.compare_exchange_weak(cur, int(t))) {}
        return;       // later tets of this chunk cannot be the lowest
      }
  });
  const int t = bad_tet.load();
  if (t == nele) return TSB_OK;
  err = "tet " + std::to_string(t) + " " + tet_problem(rest, tets + 4 * size_t(t), n);
  return TSB_E_MESH;
}

// Vertex components (union-find over the tets), numbered by their lowest vertex, with their vertices and tets in
// ascending order; vertices no tet references become orphans.
std::vector<Comp> find_components(Mesh &M, HostPlan &P) {
  UnionFind uf(M.n);
  std::vector<uint8_t> used(M.n, 0);
  for (int t = 0; t < M.nele; ++t) {
    const int32_t *v = M.tets + 4 * size_t(t);
    uf.unite(v[0], v[1]); uf.unite(v[0], v[2]); uf.unite(v[0], v[3]);
    used[v[0]] = used[v[1]] = used[v[2]] = used[v[3]] = 1;
  }
  std::vector<Comp> comps;
  std::vector<int32_t> label(M.n, -1);
  for (int v = 0; v < M.n; ++v) {
    if (!used[v]) { P.orphans.push_back(v); continue; }
    const int r = uf.find(v);
    if (label[r] < 0) { label[r] = int32_t(comps.size()); comps.emplace_back(); }
    Comp &C = comps[label[r]];
    M.local_of[v] = int32_t(C.verts.size());
    C.verts.push_back(v);
  }
  for (int t = 0; t < M.nele; ++t) comps[label[uf.find(M.tets[4 * size_t(t)])]].tets.push_back(t);
  for (Comp &C : comps) {
    for (size_t k = 0; k < C.verts.size(); ++k)
      if (C.verts[k] != C.verts[0] + int32_t(k)) { C.contiguous = 0; break; }
    P.max_comp_verts = std::max<int32_t>(P.max_comp_verts, int32_t(C.verts.size()));
    if (!C.contiguous) P.contiguous = 0;
  }
  P.n_components = int32_t(comps.size());
  return comps;
}

// Face adjacency, operator rows and staging positions of every component.  Components differ a lot in size, so
// they are handed out to the threads one at a time.
int build_components(Mesh &M, std::vector<Comp> &comps, bool identity, int nth, HostPlan &P, std::string &err) {
  std::atomic<int64_t> boundary{0};
  std::atomic<bool> bad{false};
  parallel_for(comps.size(), 1, nth, [&](size_t c0, size_t c1) {
    for (size_t c = c0; c < c1; ++c) {
      const int64_t bf = build_adjacency(M, comps[c]);
      if (bf < 0) { bad = true; continue; }
      boundary += bf;
      build_rows(M, comps[c]);
      place_vertices(comps[c], identity);
    }
  });
  if (bad) { err = "non-manifold mesh: a face is shared by more than two tets"; return TSB_E_MESH; }
  P.n_boundary_faces = int32_t(boundary.load());
  for (const Comp &C : comps) P.nnz += int64_t(C.col.size());
  return TSB_OK;
}

// Staging capacities, STAGED or GLOBAL mode (GLOBAL stores global vertex ids: identity placement, no staging) and
// the grid.
int choose_layout(std::vector<Comp> &comps, const PlanConfig &cfg, bool global_mode, HostPlan &P, std::string &err) {
  if (!global_mode) {
    int mx = 0;
    for (const Comp &C : comps) {
      mx = std::max(mx, C.npos);
      if (C.npos <= cfg.vh_cap) P.vh = std::max(P.vh, C.npos);
    }
    P.area_verts = std::max(2 * P.vh, mx);
    global_mode = mx > cfg.area_cap || mx > kMaxStagedVerts;     // colouring padded a borderline component over the cap
  }
  int G = cfg.grid;
  if (cfg.grid_cb) {
    const int rc = cfg.grid_cb(P.area_verts, global_mode, G, err);
    if (rc != TSB_OK) return rc;
  }
  if (G < 1) { err = "bad grid size"; return TSB_E_INVALID; }
  P.grid = G;
  P.mode_global = global_mode ? 1 : 0;
  if (global_mode) {
    for (Comp &C : comps) place_vertices(C, true);
    P.vh = 0; P.area_verts = 0;
  }
  return TSB_OK;
}

struct Cut { int comp; double f; };   // a point of the cost stream: fraction f of component comp

// Fills CTAs greedily up to capacity T, of which every segment a CTA opens costs F.  Returns the number of CTAs
// used and, with `out`, the cut where each of the first G begins.
int fill_ctas(const std::vector<double> &ctot, double T, double F, int G, std::vector<Cut> *out) {
  const int NC = int(ctot.size());
  int b = 0, c = 0;
  double f = 0.0;                       // position inside component c
  if (out) (*out)[0] = {0, 0.0};
  while (c < NC) {
    double cap = T - F;                 // first segment of this CTA
    while (c < NC && cap > 0) {
      const double rem = (1.0 - f) * ctot[c];
      if (rem <= cap * 1.02) {          // take the rest of the component (2% slack avoids slivers)
        cap -= rem; ++c; f = 0.0;
        if (c < NC) { cap -= F; if (cap < 0.10 * T) break; }      // not worth opening another segment
      } else {
        const double eps = std::min(0.05, 0.15 * T / std::max(ctot[c], 1e-30));
        double nf = f + cap / ctot[c];
        if (nf - f < eps) break;        // sliver: leave it to the next CTA
        if (nf > 1.0 - eps) nf = 1.0;
        f = nf; cap = 0;
        if (f >= 1.0) { ++c; f = 0.0; }
      }
    }
    ++b;
    if (out && b <= G) (*out)[b] = (c >= NC) ? Cut{NC - 1, 1.0} : Cut{c, f};
    if (b > 4 * G + 8) break;
  }
  return b;
}

// The G + 1 cuts of the cost stream (operator entries + kRowCost per row + tet_cost per tet, component after
// component); CTA b takes [cuts[b], cuts[b + 1]).  Every segment a CTA touches costs a fixed overhead F on top of
// its share of the stream (staging its component, a second set of partially filled row blocks): CTAs are filled
// up to a capacity T that includes F per segment, and T is found by bisection so that exactly G CTAs consume the
// stream.
std::vector<Cut> cut_stream(const std::vector<Comp> &comps, double tet_cost, int G) {
  const int NC = int(comps.size());
  std::vector<double> ctot(NC);
  double W = 0.0;
  for (int c = 0; c < NC; ++c) {
    const Comp &C = comps[c];
    ctot[c] = double(C.col.size()) + kRowCost * double(C.verts.size()) + tet_cost * double(C.tets.size());
    W += ctot[c];
  }
  const double F = double(kSegOverhead) * W / G;
  double lo = W / G, hi = W + F * (NC + 1) + 1.0;      // hi: one CTA could take everything
  for (int it = 0; it < 64; ++it) {
    const double mid = 0.5 * (lo + hi);
    if (fill_ctas(ctot, mid, F, G, nullptr) <= G) hi = mid; else lo = mid;
  }
  std::vector<Cut> cuts(size_t(G) + 1);
  const int used = fill_ctas(ctot, hi, F, G, &cuts);
  for (int b = std::min(used, G); b <= G; ++b) cuts[b] = {NC - 1, 1.0};   // unused CTAs (tiny meshes) get nothing
  for (int b = 1; b <= G; ++b) {   // monotone
    const Cut &a = cuts[b - 1];
    Cut &d = cuts[b];
    if (d.comp < a.comp || (d.comp == a.comp && d.f < a.f)) d = a;
  }
  return cuts;
}

struct Seg { int comp; int r0, r1, t0, t1; };   // rows [r0, r1) and tets [t0, t1) of a component

// Row of component C at fraction f of its row cost (rc: cumulative row costs, built on first use).
int row_at(const Comp &C, double f, std::vector<double> &rc) {
  const int nv = int(C.verts.size());
  if (f <= 0.0) return 0;
  if (f >= 1.0) return nv;
  if (rc.empty()) {
    rc.resize(size_t(nv) + 1, 0.0);
    for (int i = 0; i < nv; ++i) rc[i + 1] = rc[i] + double(C.rptr[i + 1] - C.rptr[i]) + kRowCost;
  }
  return int(std::lower_bound(rc.begin(), rc.end(), f * rc[nv]) - rc.begin());
}

int tet_at(const Comp &C, double f) {
  const int nt = int(C.tets.size());
  if (f <= 0.0) return 0;
  if (f >= 1.0) return nt;
  return int(std::llround(f * nt));
}

// The segments of every CTA, in CTA order (their range in P.cta_seg).
std::vector<Seg> make_segments(const std::vector<Comp> &comps, const std::vector<Cut> &cuts, HostPlan &P) {
  std::vector<Seg> segs;
  std::vector<std::vector<double>> rowcum(comps.size());
  P.cta_seg.assign(size_t(P.grid) * 2, 0);
  for (int b = 0; b < P.grid; ++b) {
    P.cta_seg[2 * size_t(b)] = int32_t(segs.size());
    const Cut lo = cuts[b], hi = cuts[b + 1];
    for (int c = lo.comp; c <= hi.comp; ++c) {
      const double f0 = (c == lo.comp) ? lo.f : 0.0, f1 = (c == hi.comp) ? hi.f : 1.0;
      if (f1 <= f0) continue;
      const Comp &C = comps[c];
      Seg s{c, row_at(C, f0, rowcum[c]), row_at(C, f1, rowcum[c]), tet_at(C, f0), tet_at(C, f1)};
      if (s.r1 <= s.r0 && s.t1 <= s.t0) continue;
      segs.push_back(s);
    }
    P.cta_seg[2 * size_t(b) + 1] = int32_t(segs.size());
  }
  return segs;
}

// Staging tables (STAGED: rest position, global id and staging position of every component vertex; GLOBAL: rest
// positions by vertex id) and the segment headers.
void staging_tables(const Mesh &M, const std::vector<Comp> &comps, const std::vector<Seg> &segs, HostPlan &P) {
  const int NC = int(comps.size());
  const bool GLOBAL = P.mode_global != 0;
  std::vector<int32_t> x4off(size_t(NC) + 1, 0), p4off(size_t(NC) + 1, 0), nseg_of(NC, 0);
  for (const Seg &g : segs) ++nseg_of[g.comp];
  if (!GLOBAL) {
    for (int c = 0; c < NC; ++c) x4off[c + 1] = x4off[c] + int32_t(comps[c].verts.size());
    P.X4.assign(size_t(x4off[NC]) * 4, 0.f);
    P.vlist.assign(size_t(x4off[NC]), 0);
    P.pos16.assign(size_t(x4off[NC]), 0);
    for (int c = 0; c < NC; ++c) p4off[c + 1] = p4off[c] + comps[c].npos;
    P.pos_gid.assign(size_t(p4off[NC]), -1);
    for (int c = 0; c < NC; ++c)
      for (size_t k = 0; k < comps[c].verts.size(); ++k) {
        const int32_t v = comps[c].verts[k];
        for (int r = 0; r < 3; ++r) P.X4[(size_t(x4off[c]) + k) * 4 + r] = M.rest[3 * size_t(v) + r];
        P.vlist[size_t(x4off[c]) + k] = v;
        P.pos16[size_t(x4off[c]) + k] = uint16_t(comps[c].pos[k]);
        P.pos_gid[size_t(p4off[c]) + comps[c].pos[k]] = v;
      }
  } else {
    P.X4.assign(size_t(M.n) * 4, 0.f);
    for (int v = 0; v < M.n; ++v)
      for (int r = 0; r < 3; ++r) P.X4[size_t(v) * 4 + r] = M.rest[3 * size_t(v) + r];
  }
  P.segs.resize(segs.size());
  for (size_t s = 0; s < segs.size(); ++s) {
    const Seg &g = segs[s];
    const Comp &C = comps[g.comp];
    SegHdr &h = P.segs[s];
    h.comp = g.comp;
    h.vbase = (GLOBAL || C.contiguous) ? (GLOBAL ? 0 : C.verts[0]) : -1;
    h.nv = int32_t(C.verts.size());
    h.x4off = GLOBAL ? C.verts[0] : x4off[g.comp];   // GLOBAL: the component's reference vertex (energy centring)
    h.expected = nseg_of[g.comp];    // one "rows stored" signal per segment (sent by the CTA's last warp)
    h.whole = (!GLOBAL && C.npos > P.vh) ? 1 : 0;
    h.npos = C.npos;
    h.p4off = GLOBAL ? 0 : p4off[g.comp];
  }
}

struct RB { int first, nrows, L, len4; };   // row block: rows[first, first + nrows), L lanes per row

// Row blocks of a segment's rows (sorted by length) that has ntc tet cells.  L lanes per row (1, 2 or 4) is chosen
// PER BLOCK: in the latency regime (the segment's cells fit the per-warp TMA rings, so nothing is ever refilled
// mid-kernel) long rows are split over adjacent lanes until a block is at most `rb_cap` quad cells, which bounds
// every warp's serial chain; in the streaming regime blocks are never split (fewest padded entries).
int row_blocks(const std::vector<RowRef> &rows, int ntc, int NW, int ring_cells, std::vector<RB> &rbs, bool &latency,
               std::string &err) {
  int64_t cells1 = ntc;                        // cells of this segment with L = 1 everywhere
  for (size_t i = 0; i < rows.size(); i += 32) cells1 += rb_len4(rows.data() + i, int(std::min<size_t>(32, rows.size() - i)), 1);
  latency = cells1 * 10 <= int64_t(ring_cells) * NW * 9;
  const int rb_cap = latency ? std::max(3, ring_cells / kRbCapDiv) : 62;
  rbs.clear();
  for (size_t i = 0; i < rows.size();) {
    int L = 1;
    while (L < kMaxLanesPerRow && rb_len4(rows.data() + i, 1, L) > rb_cap) L *= 2;
    if (rb_len4(rows.data() + i, 1, L) > 62) { err = "a vertex has more than 980 operator neighbours"; return TSB_E_MESH; }
    const int nr = int(std::min<size_t>(size_t(32 / L), rows.size() - i));
    rbs.push_back(RB{int(i), nr, L, rb_len4(rows.data() + i, nr, L)});
    i += nr;
  }
  return TSB_OK;
}

// What one CTA adds to the plan's counters, and the error that stopped it.
struct CtaStats {
  int64_t nnz_padded = 0, n_cells = 0, n_rb = 0, n_tetcells = 0, gwf[2] = {0, 0}, twf[2] = {0, 0};
  int rc = TSB_OK;
  std::string err;
};

// The streams of CTA b's warps (streams[w]; AMIPS: their rest inverses rest_inv[w]) and the CTA's entries of P.wseg.
// Row blocks (longest first) and then tet cells go to the least loaded warp; loads carry over the CTA's segments,
// which balances every warp's whole stream.
void emit_cta(const Mesh &M, const std::vector<Comp> &comps, const std::vector<Seg> &segs, int ring_cells, int b,
              HostPlan &P, std::vector<uint8_t> *streams, std::vector<float> *rest_inv, CtaStats &ES) {
  const bool GLOBAL = P.mode_global != 0;
  const int NW = P.nw;
  const int TPC = GLOBAL ? 32 : 64;                        // tets per tet cell
  const double CTC = double(kTetCellCost) * (GLOBAL ? 0.6 : 1.0);
  const int s0 = P.cta_seg[2 * size_t(b)], s1 = P.cta_seg[2 * size_t(b) + 1];
  std::vector<RowRef> rows;
  std::vector<RB> rbs;
  std::vector<int> rb_of_warp[kMaxWarps];
  LaneSlots lane_slots;
  double load[kMaxWarps] = {0};
  for (int s = s0; s < s1; ++s) {
    const Seg &g = segs[s];
    const Comp &C = comps[g.comp];
    const int32_t *gid = GLOBAL ? C.verts.data() : nullptr;
    // where this segment's component will sit in the CTA's staging area (must match the kernel:
    // "whole" components start at 0, others alternate between the two halves by position in the CTA)
    const bool whole = P.segs[s].whole != 0;
    const int ubase_bytes = GLOBAL ? 0 : (whole ? 0 : ((s - s0) & 1) * 2 * P.vh * 16);
    const int xbase_bytes = GLOBAL ? 0 : ubase_bytes + (whole ? C.npos : P.vh) * 16;
    if (!GLOBAL && xbase_bytes + C.npos * 16 > 65536) { ES.err = "internal: staging offsets exceed 16 bits"; ES.rc = TSB_E_INVALID; return; }
    rows.clear();
    for (int r = g.r0; r < g.r1; ++r) rows.push_back(RowRef{r, C.rptr[r + 1] - C.rptr[r]});
    std::stable_sort(rows.begin(), rows.end(), [](const RowRef &a, const RowRef &c) { return a.len > c.len; });
    const int ntc = (g.t1 - g.t0 + TPC - 1) / TPC;
    bool latency = false;
    if ((ES.rc = row_blocks(rows, ntc, NW, ring_cells, rbs, latency, ES.err)) != TSB_OK) return;
    const int nrb = int(rbs.size());
    for (int w = 0; w < NW; ++w) rb_of_warp[w].clear();
    {
      std::vector<int> order(nrb);
      std::iota(order.begin(), order.end(), 0);
      std::stable_sort(order.begin(), order.end(), [&](int a, int c) { return rbs[a].len4 > rbs[c].len4; });
      for (int k : order) {                  // LPT: longest block first
        int w = int(std::min_element(load, load + NW) - load);
        load[w] += double(rbs[k].len4) + (latency ? 0.0 : 0.5);
        rb_of_warp[w].push_back(k);
      }
    }
    int tc_cnt[kMaxWarps] = {0};
    const int NWT = NW > 1 ? NW - 1 : 1;     // the last warp signals "rows stored" and takes no tets (it must never wait on itself)
    for (int k = 0; k < ntc; ++k) {
      int w = int(std::min_element(load, load + NWT) - load);
      load[w] += latency ? 1.0 : CTC;        // latency regime: balance the CELL count so that every stream fits its ring
      ++tc_cnt[w];
    }
    int tnext = g.t0;
    for (int w = 0; w < NW; ++w) {
      std::vector<uint8_t> &st = streams[w];
      for (int k : rb_of_warp[w]) {
        const RB &rb = rbs[k];
        const int len4 = GLOBAL ? emit_rb<uint32_t>(st, C, rows.data() + rb.first, rb.nrows, rb.L, gid, 0, lane_slots, nullptr)
                                : emit_rb<uint16_t>(st, C, rows.data() + rb.first, rb.nrows, rb.L, nullptr, ubase_bytes, lane_slots, ES.gwf);
        ES.nnz_padded += int64_t(len4) * 4 * 32;
        ES.n_cells += len4;
      }
      for (int k = 0; k < tc_cnt[w]; ++k) {
        const int nt = std::min(TPC, g.t1 - tnext);
        std::vector<float> *bo = rest_inv ? &rest_inv[w] : nullptr;
        if (GLOBAL) emit_tc<uint32_t>(st, M, C, tnext, nt, 0, nullptr, bo);
        else emit_tc<uint16_t>(st, M, C, tnext, nt, xbase_bytes, ES.twf, bo);
        tnext += nt;
      }
      if (rb_of_warp[w].size() > 0xFFFF || tc_cnt[w] > 0xFFFF) { ES.err = "segment too large for the stream descriptors"; ES.rc = TSB_E_INVALID; return; }
      P.wseg[(size_t(s) * NW + w) * 2] = uint16_t(rb_of_warp[w].size());
      P.wseg[(size_t(s) * NW + w) * 2 + 1] = uint16_t(tc_cnt[w]);
    }
    ES.n_rb += nrb;
    ES.n_tetcells += ntc;
    ES.n_cells += ntc;
  }
}

// Every CTA's warp streams (wstream[b * nw + w]; AMIPS, when wB is not empty: the rest inverses in wB alike).
// CTAs are independent and emitted in parallel; the first failing CTA's error is reported.
int emit_ctas(const Mesh &M, const std::vector<Comp> &comps, const std::vector<Seg> &segs, int ring_cells, int nth,
              HostPlan &P, std::vector<std::vector<uint8_t>> &wstream, std::vector<std::vector<float>> &wB, std::string &err) {
  const size_t NW = size_t(P.nw);
  P.wseg.assign(segs.size() * NW * 2, 0);
  std::vector<CtaStats> stats(P.grid);
  parallel_for(size_t(P.grid), 1, nth, [&](size_t b0, size_t b1) {
    for (size_t b = b0; b < b1; ++b)
      emit_cta(M, comps, segs, ring_cells, int(b), P, &wstream[b * NW], wB.empty() ? nullptr : &wB[b * NW], stats[b]);
  });
  for (const CtaStats &e : stats) {
    if (e.rc != TSB_OK) { err = e.err; return e.rc; }
    P.nnz_padded += e.nnz_padded; P.n_cells += e.n_cells; P.n_rb += e.n_rb; P.n_tetcells += e.n_tetcells;
    P.gather_wavefronts[0] += e.gwf[0]; P.gather_wavefronts[1] += e.gwf[1];
    P.tet_wavefronts[0] += e.twf[0]; P.tet_wavefronts[1] += e.twf[1];
  }
  return TSB_OK;
}

// The plan's byte stream (the warp streams in (CTA, warp) order) and its descriptors; AMIPS: the rest inverses in
// the same order and the first tet cell of every (segment, warp).
int concat_streams(const std::vector<std::vector<uint8_t>> &wstream, const std::vector<std::vector<float>> &wB, int nth,
                   HostPlan &P, std::string &err) {
  const int G = P.grid, NW = P.nw;
  if (!wB.empty()) {
    P.wtc0.assign(P.segs.size() * NW, 0);
    const size_t per_cell = size_t(3) * (P.mode_global ? 32 : 64) * 4;
    size_t cells = 0;
    for (int b = 0; b < G; ++b)
      for (int w = 0; w < NW; ++w) {
        for (int sgi = P.cta_seg[2 * size_t(b)]; sgi < P.cta_seg[2 * size_t(b) + 1]; ++sgi) {
          P.wtc0[size_t(sgi) * NW + w] = int32_t(cells);
          cells += P.wseg[(size_t(sgi) * NW + w) * 2 + 1];
        }
        const auto &v = wB[size_t(b) * NW + w];
        P.Bt.insert(P.Bt.end(), v.begin(), v.end());
      }
    if (P.Bt.size() != cells * per_cell) { err = "internal: AMIPS rest-inverse blocks out of step with the tet cells"; return TSB_E_INVALID; }
  }
  size_t total = 0;
  for (const auto &st : wstream) total += st.size();
  if (total / 16 > 0xFFFFFFFFull) { err = "plan stream exceeds 64 GiB"; return TSB_E_NOMEM; }
  P.stream.resize(std::max<size_t>(total, 16));
  P.wdesc.assign(wstream.size() * 2, 0);
  std::vector<size_t> offs(wstream.size() + 1, 0);
  for (size_t i = 0; i < wstream.size(); ++i) {
    if (wstream[i].size() > 0xFFFFFFFFull) { err = "warp stream exceeds 4 GiB"; return TSB_E_NOMEM; }
    P.wdesc[2 * i] = uint32_t(offs[i] / 16);
    P.wdesc[2 * i + 1] = uint32_t(wstream[i].size());
    offs[i + 1] = offs[i] + wstream[i].size();
  }
  uint8_t *dst = P.stream.data();
  parallel_for(wstream.size(), 16, total > (size_t(8) << 20) ? nth : 1, [&](size_t b, size_t e) {
    for (size_t i = b; i < e; ++i)
      if (!wstream[i].empty()) std::memcpy(dst + offs[i], wstream[i].data(), wstream[i].size());
  });
  return TSB_OK;
}

}  // namespace

int build_plan(const float *rest, const int32_t *tets, int32_t n, int32_t nele, const PlanConfig &cfg,
               HostPlan &P, std::string &err) {
  if (!rest || !tets || n <= 0 || nele <= 0) { err = "null input or non-positive size"; return TSB_E_INVALID; }
  if (cfg.nw < 1 || cfg.nw > kMaxWarps || cfg.grid < 1) { err = "bad plan configuration"; return TSB_E_INVALID; }
  if (n >= 0xFFFFFF) { err = "more than 16.7 M vertices in one handle (row-block headers hold 24-bit row ids): shard the mesh"; return TSB_E_INVALID; }
  P = HostPlan();
  P.n = n; P.nele = nele; P.laplacian_scale = cfg.laplacian_scale ? 1 : 0;
  P.nw = cfg.nw;
  const int nth = std::clamp(int(std::thread::hardware_concurrency()), 1, kMaxHostThreads);

  int rc = validate(rest, tets, n, nele, nth, err);
  if (rc != TSB_OK) return rc;
  Mesh M{rest, tets, n, nele, std::vector<int32_t>(size_t(nele) * 4, -1), std::vector<int32_t>(size_t(n), -1), P.laplacian_scale};
  std::vector<Comp> comps = find_components(M, P);
  // components too large to stage keep global ids (identity placement) from the start
  const bool global_mode = cfg.force_global || P.max_comp_verts > cfg.area_cap || P.max_comp_verts > kMaxStagedVerts;
  if ((rc = build_components(M, comps, global_mode, nth, P, err)) != TSB_OK) return rc;
  if ((rc = choose_layout(comps, cfg, global_mode, P, err)) != TSB_OK) return rc;
  const std::vector<Seg> segs = make_segments(comps, cut_stream(comps, double(cfg.tet_cost), P.grid), P);
  staging_tables(M, comps, segs, P);
  std::vector<std::vector<uint8_t>> wstream(size_t(P.grid) * P.nw);
  std::vector<std::vector<float>> wB(cfg.enable_amips ? wstream.size() : 0);
  if ((rc = emit_ctas(M, comps, segs, cfg.ring_cells, nth, P, wstream, wB, err)) != TSB_OK) return rc;
  return concat_streams(wstream, wB, nth, P, err);
}

}  // namespace tsb
