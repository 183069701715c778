"""The multicolour block symmetric Gauss-Seidel preconditioner in fp64 (tsb_pcg_enable_sgs), and the host tables of the
product's builder through the test-only inspection library.  Not a test module: test_sgs_host and test_pcg_sgs import
what they use by name."""
import ctypes as C

import numpy as np

from _helpers import PLAN_DEBUG_SO

_SGS_ARRAYS = ("color", "lo_ptr", "hi_ptr", "lo", "hi", "sched", "color_ptr", "color_off", "crow", "col", "vert", "comp_off")


def sgs_tables(rest, tets, nth=0):
    """tsb::build_sgs_tables over build_hessian_pattern and build_pcg_lists of the mesh, with nth host threads (0: the
    default), as numpy arrays, plus "n_colors"."""
    lib = C.CDLL(PLAN_DEBUG_SO)
    lib.tsbdbg_sgs_build.restype = C.c_int
    lib.tsbdbg_sgs_build.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                     C.POINTER(C.c_void_p), C.POINTER(C.c_int32)]
    lib.tsbdbg_sgs_array.restype = C.c_int
    lib.tsbdbg_sgs_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
    lib.tsbdbg_sgs_free.argtypes = [C.c_void_p]
    lib.tsbdbg_last_error.restype = C.c_char_p
    rest = np.ascontiguousarray(np.asarray(rest, np.float32).reshape(-1))
    tets = np.ascontiguousarray(np.asarray(tets, np.int32).reshape(-1))
    d, nc = C.c_void_p(), C.c_int32()
    rc = lib.tsbdbg_sgs_build(rest.ctypes.data, tets.ctypes.data, rest.size // 3, tets.size // 4, 0, int(nth), C.byref(d),
                              C.byref(nc))
    if rc != 0:
        raise RuntimeError(lib.tsbdbg_last_error().decode())
    try:
        out = {"n_colors": int(nc.value)}
        for name in _SGS_ARRAYS:
            ptr, cnt = C.c_void_p(), C.c_int64()
            assert lib.tsbdbg_sgs_array(d, name.encode(), C.byref(ptr), C.byref(cnt)) == 0, name
            buf = (C.c_char * (4 * cnt.value)).from_address(ptr.value) if cnt.value else b""
            out[name] = np.frombuffer(bytes(buf), np.int32).copy()
    finally:
        lib.tsbdbg_sgs_free(d)
    return out


def block(q):
    """[6] = (xx, yy, zz, yz, xz, xy) -> symmetric [3, 3]."""
    return np.array([[q[0], q[5], q[4]], [q[5], q[1], q[3]], [q[4], q[3], q[2]]], np.float64)


def sgs_apply(A, Dinv, colors, r):
    """z = M^-1 r of one component in fp64, as the sweep forms it: A dense [3m, 3m], Dinv [m, 3, 3] the inverse diagonal
    blocks, colors [m].  Forward colour by colour, y_i = Dinv_i (r_i - sum_{col j < col i} A_ij y_j); backward, colours
    in reverse, z_i = y_i - Dinv_i sum_{col j > col i} A_ij z_j."""
    A = np.asarray(A, np.float64)
    m = len(colors)
    R = np.asarray(r, np.float64).reshape(m, 3)
    Ab = A.reshape(m, 3, m, 3).transpose(0, 2, 1, 3)           # [i, j, 3, 3]
    y = np.zeros((m, 3))
    for k in range(int(colors.max()) + 1 if m else 0):
        rows = np.flatnonzero(colors == k)
        earlier = colors < k
        s = np.einsum("ijab,jb->ia", Ab[np.ix_(rows, earlier)], y[earlier])
        y[rows] = np.einsum("iab,ib->ia", Dinv[rows], R[rows] - s)
    for k in range(int(colors.max()) if m else -1, -1, -1):
        rows = np.flatnonzero(colors == k)
        later = colors > k
        s = np.einsum("ijab,jb->ia", Ab[np.ix_(rows, later)], y[later])
        y[rows] = y[rows] - np.einsum("iab,ib->ia", Dinv[rows], s)
    return y.reshape(-1)


def sgs_matrix(A, Dinv, colors):
    """M^-1 of one component as a dense fp64 matrix (sgs_apply on the unit vectors)."""
    n3 = 3 * len(colors)
    return np.stack([sgs_apply(A, Dinv, colors, e) for e in np.eye(n3)], axis=1)


def sgs_running_bound(A, Dinv, colors, r):
    """A first-order bound of the fp32 sweep's error per entry, in units of u = 2^-24: forward zbar_i = |Dinv_i| (|r_i| +
    sum |A_ij| ybar_j), backward zbar_i = ybar_i + |Dinv_i| sum |A_ij| zbar_j (every term with its magnitude), and each
    entry's error at most (terms it sums + 3 for the block product) times the magnitude of what it sums, propagated through
    the later rows like the values themselves.  Returns (zbar, err) with err the bound on |z_fp32 - z_fp64| in units of u."""
    A = np.abs(np.asarray(A, np.float64))
    D = np.abs(np.asarray(Dinv, np.float64))
    m = len(colors)
    R = np.abs(np.asarray(r, np.float64)).reshape(m, 3)
    Ab = A.reshape(m, 3, m, 3).transpose(0, 2, 1, 3)
    nz = (Ab.reshape(m, m, 9) != 0).any(-1)
    ybar, yerr = np.zeros((m, 3)), np.zeros((m, 3))
    for k in range(int(colors.max()) + 1 if m else 0):
        rows = np.flatnonzero(colors == k)
        earlier = colors < k
        blk = Ab[np.ix_(rows, earlier)]
        n_terms = 3 * nz[np.ix_(rows, earlier)].sum(1) + 3                  # fp32 fma terms of the row, the block product
        s = R[rows] + np.einsum("ijab,jb->ia", blk, ybar[earlier])
        ybar[rows] = np.einsum("iab,ib->ia", D[rows], s)
        prop = np.einsum("iab,ib->ia", D[rows], np.einsum("ijab,jb->ia", blk, yerr[earlier]))
        yerr[rows] = (n_terms + 8)[:, None] * ybar[rows] + prop
    zbar, zerr = ybar.copy(), yerr.copy()
    for k in range(int(colors.max()) if m else -1, -1, -1):
        rows = np.flatnonzero(colors == k)
        later = colors > k
        blk = Ab[np.ix_(rows, later)]
        n_terms = 3 * nz[np.ix_(rows, later)].sum(1) + 3
        t = np.einsum("iab,ib->ia", D[rows], np.einsum("ijab,jb->ia", blk, zbar[later]))
        zbar[rows] = ybar[rows] + t
        prop = np.einsum("iab,ib->ia", D[rows], np.einsum("ijab,jb->ia", blk, zerr[later]))
        zerr[rows] = yerr[rows] + (n_terms + 8)[:, None] * t + zbar[rows] + prop
    return zbar.reshape(-1), zerr.reshape(-1)
