"""fp64 model of the affine coarse space of the per-sphere solve (tsb_pcg_enable_coarse): the closed-form coarse matrix
E_c = Z^T H Z, the basis Z, its pseudo-inverse and the two-level preconditioner P + Z E+ Z^T."""
import ctypes as C
import os

import numpy as np

from _newton_model import tet_hessians

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def coarse_tables(rest, tets):
    """The tables tsb_pcg_enable_coarse builds, through tests/native/libtsb_plan_debug.so: a dict of numpy arrays."""
    lib = C.CDLL(os.path.join(ROOT, "tests", "native", "libtsb_plan_debug.so"))
    lib.tsbdbg_coarse_build.restype = C.c_int
    lib.tsbdbg_coarse_build.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p),
                                        C.POINTER(C.c_int32)]
    lib.tsbdbg_coarse_array.restype = C.c_int
    lib.tsbdbg_coarse_array.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
    lib.tsbdbg_coarse_free.argtypes = [C.c_void_p]
    rest = np.ascontiguousarray(rest, np.float32).reshape(-1)
    tets = np.ascontiguousarray(tets, np.int32).reshape(-1)
    d, S = C.c_void_p(), C.c_int32(0)
    assert lib.tsbdbg_coarse_build(rest.ctypes.data, tets.ctypes.data, rest.size // 3, tets.size // 4, C.byref(d), C.byref(S)) == 0
    out = {"S": int(S.value)}
    try:
        for name, dt in [("tet", np.int32), ("tets", np.int32), ("B", np.float32), ("tchunk", np.int32),
                         ("comp_tchunk", np.int32), ("Y", np.float32), ("S", np.float64), ("vert", np.int32),
                         ("comp_off", np.int32), ("comp_label", np.int32)]:
            ptr, cnt = C.c_void_p(), C.c_int64(0)
            assert lib.tsbdbg_coarse_array(d, name.encode(), C.byref(ptr), C.byref(cnt)) == 0, name
            key = "Smat" if name == "S" else name
            out[key] = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(dt))), (int(cnt.value),)).copy() \
                if cnt.value else np.zeros(0, dt)
    finally:
        lib.tsbdbg_coarse_free(d)
    return out


def eps(r, s):
    return 1.0 if s == (r + 1) % 3 else -1.0


def fspace_closed_form(F, order, amips):
    """[T, 9, 9] F-space Hessians in the closed form the device's tet pass evaluates (tsb_coarse.cu): barrier on J < 0
    tets (order given, amips False) or AMIPS on J > 0 tets (amips True), unweighted."""
    T = len(F)
    Cf = np.stack([np.cross(F[:, 1], F[:, 2]), np.cross(F[:, 2], F[:, 0]), np.cross(F[:, 0], F[:, 1])], axis=1)
    J = np.einsum("tc,tc->t", F[:, 0], Cf[:, 0])
    al, be, ga, sk = (np.zeros(T) for _ in range(4))
    if amips:
        ok = J > 0
        Js = np.where(ok, J, 1.0)
        tr = (F * F).sum(axis=(1, 2))
        a = 2.0 / (3.0 * np.cbrt(Js) ** 2)
        al, be = np.where(ok, a, 0), np.where(ok, -(2.0 / 3.0) * a / Js, 0)
        ga, sk = np.where(ok, (5.0 / 9.0) * a * tr / Js ** 2, 0), np.where(ok, -a * tr / (3.0 * Js), 0)
    else:
        inv = J < 0
        m = np.where(inv, -J, 0.0)
        ga = np.where(inv, 2.0 if order == 2 else 12.0 * m * m, 0)
        sk = np.where(inv, -2.0 * m if order == 2 else -4.0 * m ** 3, 0)
    H = np.zeros((T, 9, 9))
    for a_ in range(9):
        r, c = divmod(a_, 3)
        for b_ in range(9):
            s, d = divmod(b_, 3)
            d2j = 0.0 if (r == s or c == d) else eps(r, s) * eps(c, d) * F[:, 3 - r - s, 3 - c - d]
            H[:, a_, b_] = (al * (a_ == b_) + be * (F[:, r, c] * Cf[:, s, d] + Cf[:, r, c] * F[:, s, d])
                            + ga * Cf[:, r, c] * Cf[:, s, d] + sk * d2j)
    return H


def sphere_basis(pk, s, round32=True):
    """[3 m, 9] Z of sphere s (Y = X - mean X in fp64, rounded to fp32 as the device stores it unless round32 is
    False), and Y."""
    v0, v1 = pk.vert_offsets[s], pk.vert_offsets[s + 1]
    X = pk.verts[v0:v1].astype(np.float64)
    Y = X - X.mean(0)
    if round32:
        Y = Y.astype(np.float32).astype(np.float64)
    m = v1 - v0
    Z = np.zeros((3 * m, 9))
    for r in range(3):
        for c in range(3):
            Z[r::3, 3 * r + c] = Y[:, c]
    return Z, Y


def coarse_matrices(orc, pk, x, c2, c3, order, project):
    """[S, 9, 9] sum over every sphere's tets of c2 H_b + c3 H_a in F-space (the closed form of E_c), and the per-entry
    magnitude sums sum_t |c2 H_b + c3 H_a|."""
    Hb, Ha = tet_hessians(orc, x, order, c3, project)
    Ht = c2 * Hb + c3 * Ha
    sid = np.searchsorted(pk.vert_offsets, orc.tets[:, 0], side="right") - 1
    E = np.zeros((pk.num_spheres, 9, 9))
    A = np.zeros((pk.num_spheres, 9, 9))
    np.add.at(E, sid, Ht)
    np.add.at(A, sid, np.abs(Ht))
    return E, A


def pinv_floor(E, floor):
    """E's pseudo-inverse with eigenvalues <= floor * lambda_max dropped (the zero matrix for lambda_max <= 0)."""
    w, Q = np.linalg.eigh(0.5 * (E + E.T))
    lmax = w.max()
    if not lmax > 0:
        return np.zeros_like(E)
    inv = np.where(w > floor * lmax, 1.0 / np.where(w > floor * lmax, w, 1.0), 0.0)
    return (Q * inv) @ Q.T


def shift_term(Y, mu):
    """mu (S (x) I3) in the coarse unknowns' order, S = sum Y Y^T."""
    S = Y.T @ Y
    out = np.zeros((9, 9))
    for r in range(3):
        out[3 * r:3 * r + 3, 3 * r:3 * r + 3] = mu * S
    return out


def two_level_pcg(H, b, Pinv, Z, Einv, max_iter, rtol):
    """Products of fp64 PCG with P + Z E+ Z^T to |r| <= rtol |b| (or max_iter; stops at p^T H p <= 0)."""
    M = lambda r: Pinv @ r + Z @ (Einv @ (Z.T @ r))
    x = np.zeros_like(b)
    r = b.copy()
    z = M(r)
    p = z.copy()
    rz = r @ z
    nb = np.linalg.norm(b)
    for k in range(max_iter):
        Hp = H @ p
        pHp = p @ Hp
        if pHp <= 0:
            return k + 1, False
        a = rz / pHp
        x += a * p
        r -= a * Hp
        if np.linalg.norm(r) <= rtol * nb:
            return k + 1, True
        z = M(r)
        rz_new = r @ z
        p = z + (rz_new / rz) * p
        rz = rz_new
    return max_iter, False
