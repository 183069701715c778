"""Test-side helpers: the C oracle binding, plan inspection, and a numpy emulation of the CUDA
kernel's tile algorithm (CPU checks of the host logic only -- never a product path)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
ORACLE_SO = os.path.join(ROOT, "oracle", "libtet_energy_oracle.so")


def host_has_avx2_fma() -> bool:
    try:
        flags = open("/proc/cpuinfo").read()
        return " avx2" in flags and " fma" in flags
    except OSError:
        return False


class COracle:
    """oracle/tet_energy_oracle.c through ctypes.  variant: "" = the fp64 checker; "fast" / "fast32" = the
    AVX2 timing builds (fp64 / fp32 arithmetic) used by bench.py's CPU arms only."""

    def __init__(self, rest, tets, laplacian_scale=0, variant=""):
        so = ORACLE_SO if not variant else ORACLE_SO.replace(".so", f"_{variant}.so")
        self.lib = C.CDLL(so)
        self.lib.tso_create.restype = C.c_void_p
        self.lib.tso_create.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
        self.lib.tso_destroy.argtypes = [C.c_void_p]
        self.lib.tso_energy_grad.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_int,
                                             C.c_double, C.c_void_p, C.c_void_p, C.c_int]
        self.lib.tso_energy_grad_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_double, C.c_int,
                                                C.c_double, C.c_void_p, C.c_void_p, C.c_int]
        self.rest = np.ascontiguousarray(np.asarray(rest, dtype=np.float32).reshape(-1, 3))
        self.tets = np.ascontiguousarray(np.asarray(tets, dtype=np.int32).reshape(-1, 4))
        self.n, self.nele = len(self.rest), len(self.tets)
        self.h = self.lib.tso_create(self.rest.ctypes.data, self.tets.ctypes.data, self.n, self.nele,
                                     int(laplacian_scale))
        if not self.h:
            raise ValueError("C oracle rejected the mesh")

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.tso_destroy(self.h)
            self.h = None

    def energy_grad(self, x, c1, c2, order, gradH=1.0, nthreads=0, want_grad=True):
        x = np.ascontiguousarray(np.asarray(x, dtype=np.float32).reshape(-1, 3))
        terms = np.zeros(2)
        g = np.zeros((self.n, 3)) if want_grad else None
        self.lib.tso_energy_grad(self.h, x.ctypes.data, float(c1), float(c2), int(order), float(gradH),
                                 terms.ctypes.data, g.ctypes.data if want_grad else None, int(nthreads))
        return float(c1) * terms[0] + float(c2) * terms[1], terms, g

    def energy_grad_ex(self, x, c1, c2, c3, order, gradH=1.0, nthreads=0, want_grad=True):
        """With the AMIPS term (c3): returns (total, terms[3] = smooth/barrier/amips, grad)."""
        x = np.ascontiguousarray(np.asarray(x, dtype=np.float32).reshape(-1, 3))
        terms = np.zeros(3)
        g = np.zeros((self.n, 3)) if want_grad else None
        self.lib.tso_energy_grad_ex(self.h, x.ctypes.data, float(c1), float(c2), float(c3), int(order), float(gradH),
                                    terms.ctypes.data, g.ctypes.data if want_grad else None, int(nthreads))
        return float(c1) * terms[0] + float(c2) * terms[1] + float(c3) * terms[2], terms, g


def rigid_motion(x, shift=0.0, angle=0.0, pivot_dist=5.0):
    """x (float32 [n,3]) moved rigidly in fp64, rounded once: rotated by `angle` rad about an oblique axis through a
    pivot `pivot_dist` away from the centroid, then translated by `shift` along an oblique direction."""
    x = np.asarray(x, dtype=np.float64).reshape(-1, 3)
    axis = np.array([0.3, -0.5, 0.81])
    axis /= np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    R = np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K
    pivot = x.mean(axis=0) + pivot_dist * np.array([0.6, 0.8, 0.0])
    d = np.array([1.0, -0.6, 0.3]) / np.linalg.norm([1.0, -0.6, 0.3])
    return ((x - pivot) @ R.T + pivot + shift * d).astype(np.float32)


# The moved inputs of the displacement-precision tests: (name, shift, rotation angle about a pivot 5 units away)
RIGID_MOTIONS = [("rest_pose", 0.0, 0.0), ("shift1", 1.0, 0.0), ("shift10", 10.0, 0.0), ("rot1_far_pivot", 0.0, 1.0)]


def min_abs_J(rest, tets, x):
    """Smallest |det F| over the tets at x (fp64 on the fp32 inputs)."""
    from tssplat_b200.mesh import _signed_volumes
    t = np.asarray(tets).astype(np.int64).reshape(-1, 4)
    X = np.asarray(rest, dtype=np.float32).reshape(-1, 3).astype(np.float64)
    x = np.asarray(x, dtype=np.float32).reshape(-1, 3).astype(np.float64)
    return float(np.abs(_signed_volumes(x, t) / _signed_volumes(X, t)).min())


def mirror_components(x, tets, every=2):
    """x with every `every`-th connected component mirrored through its centroid's z plane: all its tets inverted
    (J near -1) while the others keep J > 0, with |J| far from 0 (no fp32 sign flips, a well-conditioned J^(-2/3))."""
    from tssplat_b200.mesh import connected_components
    x = np.array(x, dtype=np.float32).reshape(-1, 3)
    lab = connected_components(len(x), np.asarray(tets).reshape(-1, 4))
    used = np.unique(np.asarray(tets).reshape(-1))
    for k, c in enumerate(np.unique(lab[used])):
        if k % every == 0:
            m = lab == c
            zc = x[m, 2].mean()
            x[m, 2] = 2 * zc - x[m, 2]
    return x


def pole_mesh(m):
    """One centre vertex (id 0, at the origin) with a tet to every face of the convex hull of m Fibonacci points on
    the unit sphere: the centre's operator row has m entries (the longest row the stream format must carry)."""
    from scipy.spatial import ConvexHull
    k = np.arange(m) + 0.5
    phi = np.arccos(1 - 2 * k / m)
    th = np.pi * (1 + 5 ** 0.5) * k
    P = np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], axis=1)
    f = ConvexHull(P).simplices.astype(np.int64)
    vol = np.einsum("ij,ij->i", P[f[:, 0]], np.cross(P[f[:, 1]], P[f[:, 2]]))
    f[vol < 0] = f[vol < 0][:, [0, 2, 1]]
    verts = np.concatenate([np.zeros((1, 3)), P])
    tets = np.concatenate([np.zeros((len(f), 1), np.int64), f + 1], axis=1)
    return verts, tets.astype(np.int32)


def whole_area_meshes():
    """Components staged in the whole staging area (1024..2047 positions): one alone; two mixed with 600 double-buffered
    twelve-tet spheres so that CTAs hold both kinds of segment; one of 2041 vertices that bank colouring pads past
    2047 staging positions, which sends the mesh to the global-gather mode."""
    from tssplat_b200.mesh import concat_spheres, make_pack, make_tet_sphere
    tiny = make_pack(600, 12, seed=3, unique=6)
    a, b = tiny.slice_spheres(0, 300), tiny.slice_spheres(300, 600)
    mixed = concat_spheres([(a.verts, a.tets), make_tet_sphere(1500, 7000), (b.verts, b.tets), make_tet_sphere(1501, 7700)])
    alone, near_cap = make_tet_sphere(1502, 7000), make_tet_sphere(1510, 10000)
    return {"alone": (alone[0].astype(np.float32), alone[1]), "mixed": (mixed.verts, mixed.tets),
            "near_cap": (near_cap[0].astype(np.float32), near_cap[1])}


# The meshes whose plans have shapes only they produce (assert_plan_shape says which): the 988-neighbour pole, the
# whole-area meshes and 2600 twelve-tet spheres (more segments per CTA than the shared-memory segment table holds).
PLAN_SHAPE_MESHES = ("pole", "alone", "mixed", "near_cap", "tiny2600")
_PLAN_SHAPE_CACHE = {}


def plan_shape_mesh(name):
    """(fp32 rest [n, 3], int32 tets [t, 4]) of a PLAN_SHAPE_MESHES mesh, built once."""
    if name not in _PLAN_SHAPE_CACHE:
        if name == "pole":
            V, T = pole_mesh(988)
        elif name == "tiny2600":
            from tssplat_b200.mesh import make_pack
            pk = make_pack(2600, 12, seed=3, unique=6)
            V, T = pk.verts, pk.tets
        else:
            V, T = whole_area_meshes()[name]
        _PLAN_SHAPE_CACHE[name] = (np.ascontiguousarray(V, np.float32).reshape(-1, 3),
                                   np.ascontiguousarray(T, np.int32).reshape(-1, 4))
    return _PLAN_SHAPE_CACHE[name]


def cpu_plan(sp, verts, tets, ring_slots=0, force_global=False, enable_amips=False, deterministic=False):
    """The host plan of handle sp, rebuilt on the CPU with the handle's warps and grid (and the ring it requested: row
    splitting depends on it); it must agree with the handle, so what it shows is what the kernel ran."""
    info = sp.info
    plan = build_host_plan(verts, tets, nw=info["warps_per_cta"], grid=info["grid"], force_global=int(force_global),
                           ring_slots=ring_slots, enable_amips=int(enable_amips), deterministic=int(deterministic))
    assert plan["mode_global"] == info["mode_global"] and len(plan["segs"]) == info["n_segments"]
    assert plan["nnz_padded"] == info["nnz_padded"]
    return plan


def row_blocks(plan):
    """(len4, lanes per row) of every row block in the plan's streams."""
    return [((int(h[0]) >> 24) & 63, 1 << (int(h[0]) >> 30)) for _, h in walk_streams(plan)[0]]


def segment_patterns(plan):
    """The set of per-CTA segment sequences, each segment 'whole' (whole staging area) or 'half' (double-buffered)."""
    cs = plan["cta_seg"].reshape(-1, 2)
    return {tuple("whole" if plan["segs"][s]["whole"] else "half" for s in range(a, b)) for a, b in cs if b > a}


def assert_plan_shape(name, plan, kw):
    """Fail unless the plan of a PLAN_SHAPE_MESHES mesh, built for handle options kw, has the shape that mesh is in the
    suites for: the pole's (62, 4) row block (a 62-cell row block of 4 lanes, wrapping the ring); whole-area segments
    (and for mixed a CTA with whole and double-buffered segments); near_cap in GLOBAL mode without forcing; tiny2600 at 16
    warps with more segments in one CTA than the shared-memory segment table (16) holds."""
    forced = bool(kw.get("force_global"))
    if name == "pole":
        assert (62, 4) in row_blocks(plan), "the pole's row is no longer one 62-cell row block of 4 lanes"
    elif name in ("alone", "mixed"):
        pats = segment_patterns(plan)
        assert plan["mode_global"] == 0 and any("whole" in p for p in pats), pats
        if name == "mixed":
            assert any("whole" in p and "half" in p for p in pats), pats
    elif name == "near_cap":
        assert not forced and plan["mode_global"] == 1 and plan["max_comp_verts"] <= 2047
    elif name == "tiny2600":
        cs = plan["cta_seg"].reshape(-1, 2)
        if plan["nw"] == 16:
            assert (cs[:, 1] - cs[:, 0]).max() > 16, "no CTA reads segment headers past the shared-memory table"
    else:
        raise KeyError(name)
    if forced:
        assert plan["mode_global"] == 1


# Handle options per PLAN_SHAPE_MESHES mesh, chosen to reach each shape's own paths (ring wraps of the pole's row block,
# both gather modes, both CTA widths, the register prefetch past the segment table, the deterministic gather)
PLAN_SHAPE_VARIANTS = {
    "pole": [dict(), dict(warps_per_cta=8), dict(force_global=True), dict(warps_per_cta=8, ring_slots=4),
             dict(warps_per_cta=8, force_global=True, ring_slots=4), dict(deterministic=True)],
    "alone": [dict(), dict(warps_per_cta=8), dict(deterministic=True)],
    "mixed": [dict(), dict(warps_per_cta=8), dict(deterministic=True)],
    "near_cap": [dict(), dict(warps_per_cta=8)],
    "tiny2600": [dict(), dict(warps_per_cta=8), dict(force_global=True), dict(ring_slots=3), dict(deterministic=True)],
}


def variant_id(kw):
    return "-".join(f"{a}{b}" for a, b in kw.items()) or "default"


def plan_shape_cases(deterministic=True):
    """pytest parameters (mesh, kw) over PLAN_SHAPE_VARIANTS, without the deterministic handles if not deterministic."""
    import pytest
    return [pytest.param(m, kw, id=f"{m}-{variant_id(kw)}") for m, kws in PLAN_SHAPE_VARIANTS.items() for kw in kws
            if deterministic or not kw.get("deterministic")]


def check_handle_plan_shape(name, sp, kw, enable_amips=False):
    """The CPU-rebuilt plan of handle sp (mesh name, created with options kw), checked by assert_plan_shape."""
    V, T = plan_shape_mesh(name)
    if kw.get("ring_slots"):
        assert sp.info["ring_slots"] == kw["ring_slots"], "the ring was shrunk: this variant would not test its depth"
    plan = cpu_plan(sp, V, T, ring_slots=kw.get("ring_slots", 0), force_global=kw.get("force_global", False),
                    enable_amips=enable_amips, deterministic=kw.get("deterministic", False))
    assert_plan_shape(name, plan, kw)
    return plan


PLAN_DEBUG_SO = os.path.join(ROOT, "tests", "native", "libtsb_plan_debug.so")
CELLS_PER_CHUNK = 6      # tsb_plan.h kCellsPerChunk: cells per ring slot
# Stream cells (tsb_plan.h): (cell bytes, bytes per index, tets per lane) of the STAGED (16-bit smem offsets) and
# GLOBAL (32-bit vertex ids) formats.  A cell holds 128 indices, then (at WOFF = 128 * bytes per index) 128 weights or
# the tets' 1/det(Dm); word 0 of each lane's first weight quad of a row block is the block header.
CELL_FORMAT = {False: (768, 2, 2), True: (1024, 4, 1)}
_ARRAYS = {"stream": np.uint8, "X4": np.float32, "vlist": np.int32, "segs": np.int32, "cta_seg": np.int32,
           "wdesc": np.uint32, "wseg": np.uint16, "orphans": np.int32, "pos16": np.uint16, "pos_gid": np.int32,
           "Bt": np.float32, "wtc0": np.int32, "comp_seg": np.int32, "comp_first_vertex": np.int32,
           "comp_ntets": np.int32}
_DET_ARRAYS = {"det_rowptr": np.int32, "det_vert": np.int32, "det_ent": np.uint32, "det_comp_row": np.int32,
               "det_chunk": np.int32}
_SCALARS = ("n", "nele", "n_components", "n_boundary_faces", "laplacian_scale", "mode_global", "nw", "grid", "vh",
            "area_verts", "max_comp_verts", "contiguous", "nnz", "nnz_padded", "n_rb", "n_tetcells",
            "gather_wf", "gather_wf_ideal", "tet_wf", "tet_wf_ideal")
_SEG = ("comp", "vbase", "nv", "x4off", "expected", "whole", "npos", "p4off")


def build_host_plan(rest, tets, nw=16, grid=132, laplacian_scale=0, force_global=0, vh_cap=0, area_cap=0,
                    tet_cost=0.0, ring_slots=0, enable_amips=0, deterministic=0):
    """Run the product's host plan builder (tssplat_b200/csrc/tsb_plan.cpp, no CUDA) through the
    test-only inspection library and copy its arrays out as numpy.  ring_slots: the ring a handle
    requests (row splitting depends on it); 0 = the default.  deterministic: also build (and return)
    the deterministic gather's det_* arrays."""
    lib = C.CDLL(PLAN_DEBUG_SO)
    lib.tsbdbg_build_det.restype = C.c_int
    lib.tsbdbg_build_det.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int32] * 8 + [C.c_float] + [C.c_int32] * 3 + \
                                    [C.POINTER(C.c_void_p)]
    lib.tsbdbg_array.restype = C.c_int
    lib.tsbdbg_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                 C.POINTER(C.c_int32)]
    lib.tsbdbg_scalars.argtypes = [C.c_void_p, C.c_void_p]
    lib.tsbdbg_free.argtypes = [C.c_void_p]
    lib.tsbdbg_last_error.restype = C.c_char_p
    rest = np.ascontiguousarray(np.asarray(rest, dtype=np.float32).reshape(-1))
    tets = np.ascontiguousarray(np.asarray(tets, dtype=np.int32).reshape(-1))
    d = C.c_void_p()
    rc = lib.tsbdbg_build_det(rest.ctypes.data, tets.ctypes.data, rest.size // 3, tets.size // 4, int(nw), int(grid),
                              int(laplacian_scale), int(force_global), int(vh_cap), int(area_cap), float(tet_cost),
                              int(ring_slots) * CELLS_PER_CHUNK, int(enable_amips), int(deterministic), C.byref(d))
    if rc != 0:
        raise RuntimeError(lib.tsbdbg_last_error().decode())
    try:
        plan = {}
        for name, dt in {**_ARRAYS, **(_DET_ARRAYS if deterministic else {})}.items():
            ptr, cnt, eb = C.c_void_p(), C.c_int64(), C.c_int32()
            assert lib.tsbdbg_array(d, name.encode(), C.byref(ptr), C.byref(cnt), C.byref(eb)) == 0, name
            nbytes = cnt.value * eb.value
            buf = (C.c_char * nbytes).from_address(ptr.value) if nbytes else b""
            plan[name] = np.frombuffer(bytes(buf), dtype=dt).copy()
        sc = np.zeros(20, np.int64)
        lib.tsbdbg_scalars(d, sc.ctypes.data)
        for k, v in zip(_SCALARS, sc):
            plan[k] = int(v)
    finally:
        lib.tsbdbg_free(d)
    plan["segs"] = [dict(zip(_SEG, row)) for row in plan["segs"].reshape(-1, 8).tolist()]
    return plan


def walk_streams(plan):
    """Walk every warp's cell stream as energy_grad_kernel does: CTA -> warp -> segment -> the segment's row blocks,
    then its tet cells.  Returns (blocks, cells): blocks = (byte offset, the 32 lanes' header words) of every row
    block, cells = (byte offset, CTA, segment, warp, index among the warp's tet cells of the segment) of every tet
    cell.  Asserts that each warp consumes exactly its stream."""
    G, NW = plan["grid"], plan["nw"]
    CELL, IB, _ = CELL_FORMAT[bool(plan["mode_global"])]
    WOFF = 128 * IB
    st = plan["stream"]
    wdesc, wseg, cta_seg = plan["wdesc"].reshape(G, NW, 2), plan["wseg"].reshape(-1, NW, 2), plan["cta_seg"].reshape(G, 2)
    blocks, cells = [], []
    for b in range(G):
        for w in range(NW):
            p = int(wdesc[b, w, 0]) * 16
            for s in range(cta_seg[b, 0], cta_seg[b, 1]):
                nrb, ntc = (int(v) for v in wseg[s, w])
                for _ in range(nrb):
                    hdr = st[p + WOFF:p + WOFF + 512].view(np.uint32).reshape(32, 4)[:, 0].copy()
                    blocks.append((p, hdr))
                    p += int((hdr[0] >> 24) & 63) * CELL
                for tc in range(ntc):
                    cells.append((p, b, s, w, tc))
                    p += CELL
            assert p == int(wdesc[b, w, 0]) * 16 + int(wdesc[b, w, 1]), "a warp did not consume exactly its stream"
    return blocks, cells


def tet_cell(plan, p):
    """(streamed ids [32 * TPL, 4] as int64, 1/det(Dm) [32 * TPL]) of the tet cell at byte offset p: staging byte
    offsets (STAGED) or vertex ids (GLOBAL), in slot order lane * TPL + t."""
    glob = bool(plan["mode_global"])
    _, IB, TPL = CELL_FORMAT[glob]
    n = 128 * IB * TPL
    st = plan["stream"]
    ids = st[p:p + n].view(np.uint32 if glob else np.uint16).reshape(32 * TPL, 4).astype(np.int64)
    return ids, st[p + n:p + n + 128 * TPL].view(np.float32)


def _rel_u(x, X, xr, Xr):
    """The kernel's staged displacement (rel_u in tsb_kernels.cu, the same fp32 operations): (x - X) - c with x - X
    kept exactly as a TwoSum pair, c = fp32(x_r - X_r) of the component's reference vertex r."""
    f = lambda a: np.asarray(a, dtype=np.float32)
    x, X = np.broadcast_arrays(f(x), f(X))
    c = f(xr) - f(Xr)
    s = x - X
    bb = s - x
    e = (x - (s - bb)) + (-X - bb)
    return (s - c) + e


def amips_psi(F, tr, j23):
    """The kernel's per-tet AMIPS energy psi = tr / (3 J^(2/3)) - 1 in its deviatoric form, in F's dtype: with C = F^T
    F, m = tr / 3 and D = C - m I (diagonal from differences of C's diagonal, tr D = 0), psi = (m/2 |D|^2 - det D) /
    (l (m^2 + m l + l^2)), l = j23 = J^(2/3).  F [t, 3, 3], tr and j23 [t]."""
    dt = F.dtype.type
    C = np.einsum("tri,trj->tij", F, F)
    a01, a02, a12 = C[:, 0, 0] - C[:, 1, 1], C[:, 0, 0] - C[:, 2, 2], C[:, 1, 1] - C[:, 2, 2]
    third = dt(1.0) / dt(3.0)
    d0, d1 = (a01 + a02) * third, (a12 - a01) * third
    d2 = -(d0 + d1)
    o01, o02, o12 = C[:, 0, 1], C[:, 0, 2], C[:, 1, 2]
    dd = (d0 * d0 + d1 * d1 + d2 * d2) + dt(2.0) * (o01 * o01 + o02 * o02 + o12 * o12)
    detD = d0 * (d1 * d2 - o12 * o12) - o01 * (o01 * d2 - o12 * o02) + o02 * (o01 * o12 - d1 * o02)
    m = tr * third
    return (dt(0.5) * m * dd - detD) / (j23 * (m * (m + j23) + j23 * j23))


def emulate_kernel(plan, x, c1, c2, order, gradH=1.0, dtype=np.float64, c3=None, stats=None):
    """numpy re-enactment of energy_grad_kernel (tsb_kernels.cu) on the host plan: every CTA, every
    warp walks its cell stream exactly as the kernel does (row blocks, then tet cells, segment by
    segment), with the same formulas.  Returns (energy_total, smooth, barrier, grad[n,3]); with c3
    (the AMIPS coefficient; the plan must be built with enable_amips) it also evaluates the AMIPS term of
    every J > 0 tet from the plan's per-cell rest inverses (Bt, wtc0) and returns
    (energy_total, smooth, barrier, amips, grad[n,3]).

    stats: a dict, filled with the per-sphere records of tsb_energy_grad_spheres folded per component (the plan's
    component order): "smooth", "barrier", "amips" (fp64 sums of the per-row and per-tet values), "n_inverted" (tets
    with J < 0) and "min_J" (smallest J of the component's real tets; padding tets have 1/det(Dm) = 0)."""
    if stats is not None:
        nc = plan["n_components"]
        stats.update(smooth=np.zeros(nc), barrier=np.zeros(nc), amips=np.zeros(nc),
                     n_inverted=np.zeros(nc, np.int64), min_J=np.full(nc, np.inf))
    G, NW, glob = plan["grid"], plan["nw"], bool(plan["mode_global"])
    IB = 4 if glob else 2
    idt = np.uint32 if glob else np.uint16
    CELL = 1024 if glob else 768
    TPL = 1 if glob else 2
    st = plan["stream"]
    x = np.asarray(x, dtype=np.float32).reshape(-1, 3)
    n = plan["n"]
    grad = np.full((n, 3), np.nan, dtype=dtype)
    grad[plan["orphans"]] = 0.0
    bar_add = np.zeros((n, 3), dtype=dtype)
    es = eb = ea = 0.0
    if c3 is not None:
        Bt = plan["Bt"].reshape(-1, 3, 32 * TPL, 4)                  # [tet cell][row of Dm^-1][lane * TPL + slot]
        wtc0 = plan["wtc0"].reshape(-1, NW)
        assert len(Bt) == plan["n_tetcells"], "AMIPS: one rest-inverse block per tet cell"
    X4 = plan["X4"].reshape(-1, 4)
    wdesc = plan["wdesc"].reshape(G, NW, 2)
    wseg = plan["wseg"].reshape(-1, NW, 2)
    cta_seg = plan["cta_seg"].reshape(G, 2)
    rows_done = np.zeros(plan["n_components"], dtype=np.int64)
    rows_seen = 0
    lanes = np.arange(32)
    for b in range(G):
        pos = [int(wdesc[b, w, 0]) * 16 for w in range(NW)]
        end = [pos[w] + int(wdesc[b, w, 1]) for w in range(NW)]
        assert all(int(wdesc[b, w, 1]) % CELL == 0 for w in range(NW))
        for s in range(cta_seg[b, 0], cta_seg[b, 1]):
            h = plan["segs"][s]
            nv = h["nv"]
            if glob:
                gids = np.arange(n)
                ref = X4.view(np.int32)[:, 3]                          # each vertex's reference vertex (bits in .w)
                U = _rel_u(x, X4[:, :3], x[ref], X4[ref, :3]).astype(dtype)
                Pp = x.astype(dtype)
                to_local = lambda a, base=None: a.astype(np.int64)
            else:
                vg = (h["vbase"] + np.arange(nv)) if h["vbase"] >= 0 else plan["vlist"][h["x4off"]:h["x4off"] + nv]
                npos = h["npos"]
                spos = plan["pos16"][h["x4off"]:h["x4off"] + nv].astype(np.int64)
                assert len(set(spos.tolist())) == nv and spos.max() < npos, "staging positions must be distinct"
                gids = plan["pos_gid"][h["p4off"]:h["p4off"] + npos].astype(np.int64)      # position -> global id
                assert np.array_equal(gids[spos], vg)
                U = np.full((npos, 3), np.nan, dtype=dtype)                                 # unused positions hold garbage
                Pp = np.full((npos, 3), np.nan, dtype=dtype)
                Xc = X4[h["x4off"]:h["x4off"] + nv, :3]
                U[spos] = _rel_u(x[vg], Xc, x[vg[0]], Xc[0]).astype(dtype)
                Pp[spos] = x[vg].astype(dtype)
                assert npos <= 2047 and npos <= plan["area_verts"] and (h["whole"] or npos <= plan["vh"])
                nv = npos

                li = s - cta_seg[b, 0]
                ub = 0 if h["whole"] else (li & 1) * 2 * plan["vh"]
                xb = h["npos"] if h["whole"] else ub + plan["vh"]

                def to_local(a, base=None):
                    a = a.astype(np.int64)
                    assert np.all(a % 16 == 0)
                    r = a // 16 - (ub if base is None else base)
                    assert r.min() >= 0 and r.max() < nv
                    return r
            for w in range(NW):
                nrb, ntc = (int(v) for v in wseg[s, w])
                p = pos[w]
                for _ in range(nrb):
                    acc = np.zeros((32, 3), dtype=dtype)
                    e = np.zeros(32, dtype=dtype)
                    q, len4 = 0, 1
                    while q < len4:
                        idx = to_local(st[p:p + 128 * IB].view(idt).reshape(32, 4))
                        wbits = st[p + 128 * IB:p + 128 * IB + 512].view(np.uint32).reshape(32, 4)
                        wq = wbits.view(np.float32).astype(dtype)
                        p += CELL
                        if q == 0:
                            hdr = wbits[:, 0]
                            len4 = int((hdr[0] >> 24) & 63)
                            llog = int(hdr[0] >> 30)
                            rid = (hdr & 0xFFFFFF).astype(np.int64)
                            active = rid != 0xFFFFFF
                            assert np.all(((hdr >> 24) & 63) == len4) and np.all((hdr >> 30) == llog) and 1 <= len4 <= 62
                            assert np.all(np.isfinite(wq[:, 0])), "header must read as a finite weight"
                            r = idx[:, 0]
                            ui = U[r]
                        d = U[idx] - ui[:, None, :]
                        assert np.all(d[:, 0 if q == 0 else slice(0, 0)] == 0)
                        assert np.all(wq[~active][:, 1:] == 0)
                        acc += np.einsum("lk,lkr->lr", wq, d)
                        e += np.einsum("lk,lk->l", wq, (d * d).sum(axis=2))
                        q += 1
                    L = 1 << llog
                    assert np.all(r.reshape(-1, L) == r.reshape(-1, L)[:, :1]), "the lanes of a row must be adjacent"
                    tot = acc.reshape(-1, L, 3).sum(axis=1)            # shuffle reduction over the L lanes
                    lead = (lanes % L == 0) & active
                    ra = r[lead]
                    assert np.array_equal(gids[ra], rid[lead]), "header row id must be the global id of the lane's row"
                    assert np.isnan(grad[gids[ra]]).all(), "a vertex row has two writers"
                    grad[gids[ra]] = gradH * c1 * tot[lead[::L]]
                    uref = U[h["x4off"]] if glob else U[0]
                    de = 0.5 * np.einsum("lr,lr->", ui[lead] - uref, tot[lead[::L]])
                    es += de
                    if stats is not None:
                        stats["smooth"][h["comp"]] += float(de)
                    rows_seen += int(lead.sum())
                assert ntc == 0 or w < NW - 1 or NW == 1, "the signalling warp must own no tets"
                for tc in range(ntc):
                    idx = st[p:p + 128 * IB * TPL].view(idt).reshape(32 * TPL, 4)
                    idx = to_local(idx) if glob else to_local(idx, xb)
                    idet = st[p + 128 * IB * TPL:p + 128 * IB * TPL + 128 * TPL].view(np.float32).astype(dtype)
                    p += CELL
                    q = Pp[idx]
                    e1, e2, e3 = q[:, 1] - q[:, 0], q[:, 2] - q[:, 0], q[:, 3] - q[:, 0]
                    c23 = np.cross(e2, e3)
                    J = np.einsum("lr,lr->l", e1, c23) * idet
                    inv = J < 0
                    m = np.where(inv, -J, 0.0)
                    eb += (m ** order).sum()
                    if stats is not None:
                        cp = h["comp"]
                        stats["barrier"][cp] += float((m ** order).astype(np.float64).sum())
                        stats["n_inverted"][cp] += int(inv.sum())
                        real = idet != 0                                                # padding: 1/det(Dm) = 0
                        if real.any():
                            stats["min_J"][cp] = min(stats["min_J"][cp], float(J[real].min()))
                    coef = order * m ** (order - 1)
                    k = (-coef * idet * c2 * gradH)[:, None]
                    g1, g2, g3 = k * c23, k * np.cross(e3, e1), k * np.cross(e1, e2)
                    for g, col in ((-(g1 + g2 + g3), 0), (g1, 1), (g2, 2), (g3, 3)):
                        np.add.at(bar_add, gids[idx[inv, col]], g[inv])
                    if c3 is not None:
                        # psi = tr(F^T F) / (3 J^(2/3)) - 1,  F = Ds B,  dpsi/dF = 2 / (3 J^(2/3)) (F - tr / (3 J) cof F)
                        ok = J > 0
                        B = Bt[int(wtc0[s, w]) + tc][:, ok, :3].transpose(1, 0, 2).astype(dtype)   # [tet][k][c]
                        F = np.stack([e1[ok], e2[ok], e3[ok]], axis=2) @ B                       # Ds[:, k] = e_{k+1}
                        Jp = J[ok]
                        tr = (F * F).sum(axis=(1, 2))
                        j23 = np.cbrt(Jp) ** 2
                        psi = amips_psi(F, tr, j23)
                        ea += psi.sum()
                        if stats is not None:
                            stats["amips"][h["comp"]] += float(psi.astype(np.float64).sum())
                        cof = np.linalg.det(F)[:, None, None] * np.linalg.inv(F).transpose(0, 2, 1)
                        P = (2 / (3 * j23) * c3 * gradH)[:, None, None] * (F - (tr / (3 * Jp))[:, None, None] * cof)
                        gk = P @ B.transpose(0, 2, 1)                                             # [tet][r][k]: vertex k+1
                        for k in range(3):
                            np.add.at(bar_add, gids[idx[ok, k + 1]], gk[:, :, k])
                        np.add.at(bar_add, gids[idx[ok, 0]], -gk.sum(axis=2))
                pos[w] = p
            rows_done[h["comp"]] += 1
        assert pos == end, "a warp did not consume exactly its stream"
    for sg in plan["segs"]:
        assert rows_done[sg["comp"]] == sg["expected"], "rows-done counter would never reach `expected`"
    assert rows_seen == n - len(plan["orphans"]) and not np.isnan(grad).any()
    if c3 is not None:
        return c1 * es + c2 * eb + c3 * ea, es, eb, ea, grad + bar_add
    return c1 * es + c2 * eb, es, eb, grad + bar_add
