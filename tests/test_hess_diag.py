"""Per-vertex 3x3 diagonal blocks of the geometry-energy Hessian (tsb_hess_diag, TetSpheres.hess_diag,
SmoothnessBarrierEnergy.hess_diag) and the block-Jacobi helpers of tssplat_b200.newton.

CPU: an fp64 reference in matrix form on the oracle's G and M (G_k^T Hess(psi) G_k per tet corner, M's diagonal blocks)
against central differences of the oracle's gradient, known answers (rest, uniform scale, rotation, rank-1 PSD barrier
blocks, the smoothness part), a re-enactment of the kernel's row pass on the streamed plan (with a mutation that counts
the header slot), an fp32 re-enactment of the tet blocks that calibrates the per-row bound of the GPU checks, and
block_jacobi.  GPU: the kernel against the fp64 reference per row, a cross-check against tsb_hvp_ex, gradH scaling,
bitwise repeatability, chaining, handle info, argument errors, and preconditioned CG end to end."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp

from _helpers import (CELL_FORMAT, build_host_plan, check_handle_plan_shape, min_abs_J, mirror_components, plan_shape_cases,
                      walk_streams)
from oracle.tet_energy_oracle import ReferenceEnergyOracle, _cof3, _det3, rest_inverse
from test_hvp import _cof_pair
from tssplat_b200.mesh import make_pack, perturb

U = 2.0 ** -24            # fp32 unit roundoff
KAPPA = 64                # per-row bound |D - D64| <= KAPPA u A_i (calibrated by test_fp32_reenactment_within_bound)
GH = 0.7                  # gradH of the GPU runs
C3 = 0.5                  # AMIPS coefficient of the c3 != 0 runs


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference, in matrix form.  vec F_t = G_t x (row-major), so moving corner k of tet t moves vec F_t by G_{t,k}
# (9 x 3) and the corner's diagonal block of the tet term is G_{t,k}^T Hess(psi)(F_t) G_{t,k}, with the 9 x 9 Hessian of
# psi assembled column by column from its directional derivative dP[dF] (the derivative of dpsi/dF along dF):
#     barrier, psi = max(-J, 0)^p:   dP = phi''(J) (C : dF) C + phi'(J) dC,   dC = cof_pair(F, dF) + cof_pair(dF, F)
#     AMIPS,   psi = I1 / (3 J^(2/3)) - 1 (J > 0):   dP = da (F - beta C) + a (dF - dbeta C - beta dC)
# The smoothness part is c1 times the 3 x 3 diagonal block of M = G^T L^T L G.


def corner_G(orc):
    """[T, 4, 9, 3]: d vec(F_t) / d x_{v_k} of every tet corner k, read from the oracle's G."""
    if not hasattr(orc, "_corner_G"):
        G = orc.G.tocoo()
        t, m, v, s = G.row // 9, G.row % 9, G.col // 3, G.col % 3
        k = np.argmax(orc.tets[t] == v[:, None], axis=1)
        out = np.zeros((orc.nele, 4, 9, 3))
        np.add.at(out, (t, k, m, s), G.data)
        orc._corner_G = out
    return orc._corner_G


def psi_hessians(F, order=None, amips=False):
    """[T, 9, 9] Hessians of the barrier (order given) or of AMIPS (amips=True) with respect to vec F."""
    T = len(F)
    J = _det3(F)
    C = _cof3(F)
    tr = (F * F).sum(axis=(1, 2))
    inv, ok = J < 0, J > 0
    m = np.where(inv, -J, 0.0)
    if order is not None:
        d1, d2 = -order * m ** (order - 1), order * (order - 1) * m ** (order - 2)
    Js = np.where(ok, J, 1.0)
    a = 2.0 / (3.0 * Js ** (2.0 / 3.0))
    beta = tr / (3.0 * Js)
    e = lambda s: s[:, None, None]
    H = np.zeros((T, 9, 9))
    for q in range(9):
        dF = np.zeros_like(F)
        dF[:, q // 3, q % 3] = 1.0
        dJ = np.einsum("tij,tij->t", C, dF)
        dC = _cof_pair(F, dF) + _cof_pair(dF, F)
        if amips:
            da = -2.0 / 3.0 * a * dJ / Js
            dbeta = 2.0 * np.einsum("tij,tij->t", F, dF) / (3.0 * Js) - tr * dJ / (3.0 * Js ** 2)
            dP = e(da) * (F - e(beta) * C) + e(a) * (dF - e(dbeta) * C - e(beta) * dC)
            dP[~ok] = 0
        else:
            dP = e(d2 * dJ) * C + e(d1) * dC
            dP[~inv] = 0
        H[:, :, q] = dP.reshape(T, 9)
    return H


def tet_hessians(V, T, x, c2, c3, order, project=False, rest64=False):
    """[T, 12, 12] per tet: K_t^T (c2 H_b + c3 H_a) K_t and its magnitude c2 |K_t^T H_b K_t| + c3 |K_t^T H_a K_t|
    (corner-major, three coordinates per corner), on the kernels' inputs: F = E B with B = fp32 Dm^-1 (fp64 with
    rest64) and corner vectors from B, E the exact edges of the fp32 x, or with project the fp32-rounded edges the
    projection forms and each term's 9 x 9 Hessian projected to PSD.  An AMIPS tet's Hessian grows like I1 / J^2, so a
    relative rounding of an edge moves it by far more than u A_ij on a near-flat tet: the kernels' own roundings of their
    inputs are not what the checks built on this measure."""
    T = np.asarray(T, np.int64).reshape(-1, 4)
    B = rest_inverse(V, T)
    if not rest64:
        B = B.astype(np.float32).astype(np.float64)
    x32 = np.asarray(x, np.float32).reshape(-1, 3)
    if project:
        E = np.stack([(x32[T[:, k]] - x32[T[:, 0]]).astype(np.float64) for k in (1, 2, 3)], 1)
    else:
        E = np.stack([x32[T[:, k]].astype(np.float64) - x32[T[:, 0]].astype(np.float64) for k in (1, 2, 3)], 1)
    F = np.einsum("tkr,tkc->trc", E, B)
    a = np.concatenate([-B.sum(axis=1, keepdims=True), B], axis=1)            # [T, 4, 3]
    Km = np.zeros((len(T), 9, 12))
    for k in range(4):
        for r in range(3):
            Km[:, 3 * r:3 * r + 3, 3 * k + r] = a[:, k]
    H, A = np.zeros((len(T), 12, 12)), np.zeros((len(T), 12, 12))
    for wgt, kind in ((c2, dict(order=order)), (c3, dict(amips=True))):
        if not wgt:
            continue
        Hm = psi_hessians(F, **kind)
        if project:
            w, Q = np.linalg.eigh(0.5 * (Hm + Hm.transpose(0, 2, 1)))
            Hm = np.einsum("tij,tj,tkj->tik", Q, np.maximum(w, 0), Q)
        Kt = wgt * np.einsum("tma,tmn,tnb->tab", Km, Hm, Km, optimize=True)
        H += Kt
        A += np.abs(Kt)
    return H, A


def corner_blocks(orc, x, order=None, amips=False):
    """[T, 4, 3, 3]: the diagonal block of every tet corner of one tet term at x."""
    F = (orc.G @ np.asarray(x, np.float64).reshape(-1)).reshape(-1, 3, 3)
    Gk = corner_G(orc)
    return np.einsum("tkma,tmn,tknb->tkab", Gk, psi_hessians(F, order, amips), Gk, optimize=True)


def smooth_blocks(orc):
    """[n, 3, 3]: the diagonal blocks of M."""
    i = np.arange(orc.n)
    D = np.zeros((orc.n, 3, 3))
    for r in range(3):
        for s in range(3):
            D[:, r, s] = np.asarray(orc.M[3 * i + r, 3 * i + s]).ravel()
    return D


def scatter(orc, blk):
    D = np.zeros((orc.n, 3, 3))
    np.add.at(D, orc.tets, blk)
    return D


def hess_diag_blocks(orc, x, c1, c2, c3, order):
    """[n, 3, 3]: the diagonal blocks D_i of H(x) = c1 M + c2 sum_t H_t + c3 sum_t H_a,t."""
    D = c1 * smooth_blocks(orc) + c2 * scatter(orc, corner_blocks(orc, x, order=order))
    if c3:
        D = D + c3 * scatter(orc, corner_blocks(orc, x, amips=True))
    return D


def magnitudes(orc, x, order):
    """Per-vertex magnitude forms (sum_j |M_ij|, barrier, AMIPS), each [n]: the terms of A_i in the per-row bound,
    sums over the vertex's tet corners of p (p-1) m^(p-2) |g|^2 and a (|b|^2 + 4 |g| |f| / (3J) + 5 I1 |g|^2 / (9 J^2))
    (g = C b, f = F b, b the corner's column of G: the closed form's three terms taken in absolute value)."""
    M1 = abs(orc.M[0::3, 0::3])
    sm = np.asarray(M1.sum(axis=1)).ravel()
    F = (orc.G @ np.asarray(x, np.float64).reshape(-1)).reshape(-1, 3, 3)
    J = _det3(F)
    Cf = _cof3(F)
    tr = (F * F).sum(axis=(1, 2))
    b = corner_G(orc)[:, :, 0:3, 0]                                    # [T, 4, 3]: b_k
    g = np.linalg.norm(np.einsum("trc,tkc->tkr", Cf, b), axis=2)
    f = np.linalg.norm(np.einsum("trc,tkc->tkr", F, b), axis=2)
    m = np.where(J < 0, -J, 0.0)
    bar = (order * (order - 1) * m ** (order - 2) * (J < 0))[:, None] * g * g
    ok = J > 0
    Js = np.where(ok, J, 1.0)
    a = 2.0 / (3.0 * Js ** (2.0 / 3.0))
    am = (a * ok)[:, None] * ((b * b).sum(axis=2) + 4.0 * g * f / (3.0 * Js[:, None]) + 5.0 * tr[:, None] * g * g / (9.0 * Js[:, None] ** 2))
    out = []
    for v in (bar, am):
        s_ = np.zeros(orc.n)
        np.add.at(s_, orc.tets, v)
        out.append(s_)
    return sm, out[0], out[1]


def planes_of(D):
    """[n, 3, 3] -> the [2, n, 3] layout of tsb_hess_diag."""
    return np.stack([np.stack([D[:, 0, 0], D[:, 1, 1], D[:, 2, 2]], 1), np.stack([D[:, 1, 2], D[:, 0, 2], D[:, 0, 1]], 1)])


def coloring(orc):
    """Vertex classes with no shared M entry and no shared tet (greedy, in vertex order)."""
    A = (abs(orc.M[0::3, 0::3]) > 0).astype(np.int8)
    t = orc.tets
    rows = np.repeat(t, 4, axis=1).ravel()
    cols = np.tile(t, (1, 4)).ravel()
    A = (A + sp.csr_matrix((np.ones(rows.size, np.int8), (rows, cols)), shape=A.shape)).tocsr()
    col = np.full(orc.n, -1)
    for i in range(orc.n):
        used = set(col[A.indices[A.indptr[i]:A.indptr[i + 1]]].tolist())
        c = 0
        while c in used:
            c += 1
        col[i] = c
    return [np.nonzero(col == c)[0] for c in range(col.max() + 1)]


# ---------------------------------------------------------------------------------------------------------------------
# CPU


@pytest.fixture(scope="module")
def small():
    pk = make_pack(3, 512, seed=4)
    orc = ReferenceEnergyOracle(pk.verts, pk.tets)
    xs = {"benign": perturb(pk, sigma_rel=0.1, seed=1), "mirrored": mirror_components(perturb(pk, sigma_rel=0.1, seed=2), pk.tets)}
    for x in xs.values():
        assert min_abs_J(pk.verts, pk.tets, x) > 1e-2
    return SimpleNamespace(pk=pk, orc=orc, x={k: v.astype(np.float64) for k, v in xs.items()}, classes=coloring(orc))


def _fd_blocks(orc, x, c1, c2, c3, order, classes, eps=2e-6):
    """Central differences of the oracle's gradient along v = sum_{i in S} e_{3i+a} per vertex class S, Richardson-
    extrapolated from steps eps and eps / 2 (the edges are ~1e-2 long, so the plain difference's (eps / h)^2 term would
    dominate the comparison)."""
    g = lambda y: orc.backward(1.0, y, c1, c2, order) + orc.amips_backward(1.0, y, c3)
    D = np.zeros((orc.n, 3, 3))
    for S in classes:
        for a in range(3):
            v = np.zeros((orc.n, 3))
            v[S, a] = 1.0
            cd = lambda h: ((g(x + h * v) - g(x - h * v)) / (2 * h)).reshape(-1, 3)
            fd = (4.0 * cd(eps / 2) - cd(eps)) / 3.0
            D[S, :, a] = fd[S]
    return D


@pytest.mark.parametrize("c3", [0.0, 0.7], ids=["no-amips", "amips"])
@pytest.mark.parametrize("order", [2, 4])
@pytest.mark.parametrize("case", ["benign", "mirrored"])
def test_reference_matches_central_differences(small, case, order, c3):
    orc, x = small.orc, small.x[case]
    c1, c2 = 1e-3, 1.0
    D = hess_diag_blocks(orc, x, c1, c2, c3, order)
    fd = _fd_blocks(orc, x, c1, c2, c3, order, small.classes)
    scale = np.abs(D).max(axis=(1, 2))
    err = np.abs(D - fd).max(axis=(1, 2))
    assert (err <= 1e-8 * scale + 1e-10 * scale.max()).all(), (err / scale).max()
    if case == "mirrored":
        assert np.abs(scatter(orc, corner_blocks(orc, x, order=order))).max() > 0


def test_known_answers_at_rest(small):
    """At x = X every F = I: no barrier, and the AMIPS block of a corner is (2/3)(|b|^2 I + b b^T / 3)."""
    orc, pk = small.orc, small.pk
    X = pk.verts.astype(np.float32).astype(np.float64)
    B = rest_inverse(X, pk.tets)
    b = np.concatenate([-B.sum(axis=1, keepdims=True), B], axis=1)          # [T, 4, 3]: b_k
    expect = 2.0 / 3.0 * ((b * b).sum(axis=2)[:, :, None, None] * np.eye(3) + np.einsum("tka,tkb->tkab", b, b) / 3.0)
    D = hess_diag_blocks(orc, X, 0.0, 0.0, 1.0, 2)
    ref = scatter(orc, expect)
    assert np.abs(D - ref).max() <= 1e-9 * np.abs(ref).max()
    assert not scatter(orc, corner_blocks(orc, X, order=2)).any()


def test_known_answers_scale_and_rotation(small):
    """AMIPS blocks scale as s^-2 under x -> s x; every term's block becomes R D R^T under x -> R x."""
    orc = small.orc
    x = small.x["benign"]
    Da = hess_diag_blocks(orc, x, 0.0, 0.0, 1.0, 2)
    for s in (0.5, 3.0):
        assert np.abs(hess_diag_blocks(orc, s * x, 0.0, 0.0, 1.0, 2) - Da / s ** 2).max() <= 1e-9 * np.abs(Da).max() / s ** 2
    th = 0.7
    R = np.array([[np.cos(th), -np.sin(th), 0.0], [np.sin(th), np.cos(th), 0.0], [0.0, 0.0, 1.0]])
    R = R @ np.array([[1.0, 0.0, 0.0], [0.0, np.cos(0.3), -np.sin(0.3)], [0.0, np.sin(0.3), np.cos(0.3)]])
    for case in ("benign", "mirrored"):
        x = small.x[case]
        for order in (2, 4):
            D = hess_diag_blocks(orc, x, 1e-3, 1.0, 0.7, order)
            Dr = hess_diag_blocks(orc, x @ R.T, 1e-3, 1.0, 0.7, order)
            assert np.abs(Dr - R @ D @ R.T).max() <= 1e-9 * np.abs(D).max()


def test_barrier_blocks_rank1_psd_and_smoothness_part(small):
    orc = small.orc
    x = small.x["mirrored"]
    for order in (2, 4):
        blk = corner_blocks(orc, x, order=order).reshape(-1, 3, 3)
        lam = np.linalg.eigvalsh(blk)
        top = np.abs(lam).max(axis=1, keepdims=True)
        assert (lam[:, 2:] >= 0).all() and (np.abs(lam[:, :2]) <= 1e-12 * np.maximum(top, 1e-300)).all()
        assert (lam[:, 2] > 0).sum() > 0
    Ds = hess_diag_blocks(orc, x, 0.3, 0.0, 0.0, 2)
    Mii = orc.M.diagonal()[0::3]
    assert np.array_equal(Ds, 0.3 * Mii[:, None, None] * np.eye(3))
    assert np.array_equal(orc.M.diagonal()[1::3], Mii) and np.array_equal(orc.M.diagonal()[2::3], Mii)


def row_pass(plan, include_header=False):
    """The DIAG row pass re-enacted on the streamed plan, in fp32: for every row, minus the sum of its streamed weights
    whose column is not the row itself (each lane's header slot has the row as its column).  {global row id: M_ii}."""
    glob = bool(plan["mode_global"])
    CELL, IB, _ = CELL_FORMAT[glob]
    WOFF = 128 * IB
    idt = np.uint32 if glob else np.uint16
    st = plan["stream"]
    blocks, _ = walk_streams(plan)
    out = {}
    for p, hdr in blocks:
        len4, llog = int((hdr[0] >> 24) & 63), int(hdr[0] >> 30)
        rid = (hdr & 0xFFFFFF).astype(np.int64)
        rowj = st[p:p + 128 * IB].view(idt).reshape(32, 4)[:, 0]
        acc = np.zeros(32, np.float32)
        for q in range(len4):
            base = p + q * CELL
            j = st[base:base + 128 * IB].view(idt).reshape(32, 4)
            w = st[base + WOFF:base + WOFF + 512].view(np.float32).reshape(32, 4)
            keep = np.ones_like(w, bool) if include_header else j != rowj[:, None]
            for c in range(4):
                acc = (acc + np.where(keep[:, c], w[:, c], np.float32(0))).astype(np.float32)
        L = 1 << llog
        tot = acc.reshape(-1, L).sum(axis=1, dtype=np.float32)
        for r in range(32 // L):
            if rid[r * L] != 0xFFFFFF:
                assert int(rid[r * L]) not in out, "a row has two writers"
                out[int(rid[r * L])] = -float(tot[r])
    return out


@pytest.mark.parametrize("force_global", [0, 1], ids=["staged", "global"])
def test_row_pass_reenactment(small, force_global):
    """The weight sum of every row gives M_ii within KAPPA u sum_j |M_ij|; counting the header slot does not."""
    orc, pk = small.orc, small.pk
    plan = build_host_plan(pk.verts, pk.tets, force_global=force_global)
    Mii = orc.M.diagonal()[0::3]
    A = np.asarray(abs(orc.M[0::3, 0::3]).sum(axis=1)).ravel()
    got = row_pass(plan)
    assert sorted(got) == list(range(orc.n))
    ids = np.array(sorted(got))
    d = np.array([got[i] for i in ids])
    ratio = np.abs(d - Mii[ids]) / (U * A[ids])
    print(f"row pass: max |M_ii - fp32 sum| / (u sum|M_ij|) = {ratio.max():.3g}")
    assert ratio.max() <= KAPPA / 4
    bad = row_pass(plan, include_header=True)
    dbad = np.array([bad[i] for i in ids])
    assert (~(np.abs(dbad - Mii[ids]) <= KAPPA * U * A[ids])).any()


def fp32_tet_blocks(V, T, x, order, c2, c3):
    """The kernel's tet blocks in fp32 per tet (cross products of the fp32 edges times fp32 1/det(Dm), F = Ds B with
    fp32 B, the closed form), summed into fp32 rows in tet order: [n, 3, 3]."""
    f32 = np.float32
    T = np.asarray(T, np.int64)
    B = rest_inverse(V, T).astype(f32)
    Xd = np.asarray(V, np.float32).astype(np.float64)[T]
    idet = (1.0 / np.linalg.det(np.transpose(Xd[:, 1:] - Xd[:, :1], (0, 2, 1)))).astype(f32)
    P = np.asarray(x, f32)[T]
    e1, e2, e3 = (P[:, k] - P[:, 0] for k in (1, 2, 3))
    J = (e1 * np.cross(e2, e3)).sum(axis=1, dtype=f32) * idet
    inv, ok = J < 0, (J > 0) & (c3 != 0)
    m = np.where(inv, -J, f32(0))
    ga = np.where(inv, f32(c2) * (f32(2) if order == 2 else f32(12) * m * m), f32(0))
    al = np.zeros_like(J)
    be = np.zeros_like(J)
    Fm = np.einsum("tkr,tkc->trc", np.stack([e1, e2, e3], 1), B).astype(f32)
    Js = np.where(ok, J, f32(1))
    tr = (Fm * Fm).sum(axis=(1, 2), dtype=f32)
    cb = np.cbrt(Js).astype(f32)
    a = f32(c3) * (f32(2) / (f32(3) * (cb * cb)))
    iJ = f32(1) / Js
    al = np.where(ok, a, al)
    be = np.where(ok, -f32(2 / 3) * a * iJ, be)
    ga = np.where(ok, f32(5 / 9) * a * tr * (iJ * iJ), ga)
    bk_all = [-(B[:, 0] + B[:, 1] + B[:, 2]), B[:, 0], B[:, 1], B[:, 2]]
    ck = [np.cross(e3 - e1, e2 - e1), np.cross(e2, e3), np.cross(e3, e1), np.cross(e1, e2)]
    D = np.zeros((len(V), 3, 3), f32)
    act = inv | ok
    for k in range(4):
        g = (idet[:, None] * ck[k]).astype(f32)
        f = np.einsum("trc,tc->tr", Fm, bk_all[k]).astype(f32)
        f = np.where(ok[:, None], f, f32(0))
        b2 = np.where(ok, (bk_all[k] * bk_all[k]).sum(axis=1, dtype=f32), f32(0))
        blk = (al * b2)[:, None, None] * np.eye(3, dtype=f32) + be[:, None, None] * (
            g[:, :, None] * f[:, None, :] + f[:, :, None] * g[:, None, :]) + ga[:, None, None] * g[:, :, None] * g[:, None, :]
        blk[~act] = 0
        np.add.at(D, T[:, k], blk.astype(f32))
    return D


def test_fp32_reenactment_within_bound(small):
    """The per-row bound |D - D64|_max <= KAPPA u A_i of the GPU checks holds for the fp32 re-enactment of the rows
    (row_pass) and the tet blocks with room to spare."""
    orc, pk = small.orc, small.pk
    plan = build_host_plan(pk.verts, pk.tets)
    rows = row_pass(plan)
    Mii32 = np.array([rows[i] for i in range(orc.n)], np.float32)
    worst = 0.0
    for case, x in small.x.items():
        for order in (2, 4):
            for c1, c2, c3 in ((1e-3, 1.0, 0.0), (1e-3, 1.0, C3), (0.0, 1.0, C3)):
                D64 = hess_diag_blocks(orc, x, c1, c2, c3, order)
                D32 = fp32_tet_blocks(pk.verts, pk.tets, x, order, c2, c3)
                D32 = D32 + (np.float32(c1) * Mii32)[:, None, None] * np.eye(3, dtype=np.float32)
                sm, bar, am = magnitudes(orc, x, order)
                A = c1 * sm + c2 * bar + c3 * am
                r = (np.abs(D32.astype(np.float64) - D64).max(axis=(1, 2)) / (U * A)).max()
                worst = max(worst, r)
    print(f"fp32 re-enactment: max |D - D64| / (u A_i) = {worst:.3g} (KAPPA {KAPPA})")
    assert worst <= KAPPA / 4


def test_block_jacobi():
    import torch
    from tssplat_b200.newton import block_jacobi, hess_blocks
    rng = np.random.default_rng(3)
    Q = np.linalg.qr(rng.normal(size=(6, 3, 3)))[0]
    lam = np.array([[1.0, 2.0, 5.0], [1e-3, 1.0, 4.0], [-2.0, 1.0, 3.0], [-1.0, -0.5, -0.1], [0.0, 0.0, 0.0], [0.0, 0.0, 2.0]])
    D = np.einsum("nij,nj,nkj->nik", Q, lam, Q)
    D[4] = 0.0
    P = block_jacobi(torch.from_numpy(planes_of(D)), rel_floor=1e-2).numpy()
    assert np.allclose(hess_blocks(torch.from_numpy(planes_of(D))).numpy(), D, atol=1e-14)
    # SPD blocks: the inverse (the floor 1e-2 * 5 = 0.05 clamps nothing in block 0)
    assert np.allclose(P[0], np.linalg.inv(D[0]), rtol=1e-10, atol=1e-12)
    for i in (0, 1, 2, 5):
        w = np.linalg.eigvalsh(P[i])
        assert np.allclose(P[i], P[i].T) and (w > 0).all()
    # the floor applies to small and negative eigenvalues: 1e-3 -> 0.04, -2 -> 0.03, 0 -> 0.02
    for i, floored in ((1, [0.04, 1.0, 4.0]), (2, [0.03, 1.0, 3.0]), (5, [0.02, 0.02, 2.0])):
        expect = np.einsum("ij,j,kj->ik", Q[i], 1.0 / np.maximum(lam[i], max(floored[0], 1e-2 * lam[i].max())), Q[i])
        assert np.allclose(P[i], expect, rtol=1e-9, atol=1e-12), i
    # lambda_max <= 0 and zero blocks map to 0
    assert not P[3].any() and not P[4].any()


# ---------------------------------------------------------------------------------------------------------------------
# GPU


def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch


@pytest.fixture(scope="module")
def ext():
    _torch()
    from tssplat_b200 import tet_spheres_ext
    return tet_spheres_ext


def _handle(ext, V, T, **kw):
    return ext.TetSpheres(np.ascontiguousarray(V, np.float32).reshape(-1), np.ascontiguousarray(T, np.int32).reshape(-1), **kw)


_REFS = {}


def _refs(mesh):
    """(rest, tets, oracle, {case: (x, smooth blocks, {order: barrier blocks}, AMIPS blocks, magnitudes)}): the meshes
    and inputs of tests/test_hvp_amips.py (every |J| > 0.05, so fp32 and fp64 agree on the active sets)."""
    if mesh not in _REFS:
        from test_hvp_amips import _mesh
        V, T, orc, inputs, _ = _mesh(mesh)
        Ds = smooth_blocks(orc)
        cases = {}
        for case, (x, _) in inputs.items():
            x64 = x.astype(np.float64)
            Db = {o: scatter(orc, corner_blocks(orc, x64, order=o)) for o in (2, 4)}
            Da = scatter(orc, corner_blocks(orc, x64, amips=True))
            mags = {o: magnitudes(orc, x64, o) for o in (2, 4)}
            cases[case] = (x, Db, Da, mags)
        _REFS[mesh] = (V, T, orc, Ds, cases)
    return _REFS[mesh]


def _check_against_fp64(sp, mesh, key_prefix, orphans=None):
    torch = _torch()
    V, T, orc, Ds, cases = _refs(mesh)
    active = 0
    for case, (x, Db, Da, mags) in cases.items():
        xt = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
        for order in (2, 4):
            sm, bar, am = mags[order]
            for c1, c2, c3 in ((2e-3, 0.8, 0.0), (2e-3, 0.8, C3)):
                key = (key_prefix, case, order, c3)
                got = sp.hess_diag(xt, c1, c2, order, c3=c3, gradH=GH).cpu().numpy().astype(np.float64)
                D = c1 * Ds + c2 * Db[order] + c3 * Da
                err = np.abs(got - GH * planes_of(D)).max(axis=(0, 2))
                A = GH * (c1 * sm + c2 * bar + c3 * am)
                assert (err <= KAPPA * U * A).all(), (key, (err / (U * A)).max())
                if orphans is not None:
                    assert not got[:, orphans].any(), key
                active += int(np.abs(Db[order]).max() > 0)
    assert active > 0


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(warps_per_cta=8), dict(deterministic=True),
                                dict(warps_per_cta=8, deterministic=True)],
                         ids=["w16", "w8", "w16-det", "w8-det"])
def test_hess_diag_staged_pack(ext, kw):
    V, T, *_ = _refs("pack64x4096")
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    assert sp.info["mode_global"] == 0
    _check_against_fp64(sp, "pack64x4096", str(kw))


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(force_global=True), dict(force_global=True, warps_per_cta=8, deterministic=True)],
                         ids=["global", "global-w8-det"])
def test_hess_diag_a_veg_global(ext, kw):
    V, T, *_ = _refs("a_veg")
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    assert sp.info["mode_global"] == 1
    _check_against_fp64(sp, "a_veg", str(kw))


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(force_global=True), dict(warps_per_cta=8, ring_slots=3, deterministic=True)],
                         ids=["staged", "global", "w8-ring3-det"])
def test_hess_diag_shuffled_ids_with_orphans(ext, kw):
    V, T, *_ = _refs("shuffled")
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    orphans = np.ones(len(V), bool)
    orphans[np.unique(T)] = False
    assert orphans.sum() == 500
    _check_against_fp64(sp, "shuffled", str(kw), orphans=orphans)


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
def test_cross_check_against_hvp(ext, det):
    """For v = sum_{i in S} e_{3i+a} over a vertex set S with no shared M entry and no shared tet, (H v)_i is column a of
    D_i: tsb_hvp_ex and tsb_hess_diag agree there within the per-row bound."""
    torch = _torch()
    V, T, orc, Ds, cases = _refs("shuffled")
    sp = _handle(ext, V, T, enable_amips=True, deterministic=det)
    classes = [S for S in coloring(orc) if len(S)]
    c1, c2 = 2e-3, 0.8
    for case in ("inverted_o2", "stretched_o2"):
        x = cases[case][0]
        sm, bar, am = cases[case][3][4]
        A = c1 * sm + c2 * bar + C3 * am
        xt = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
        planes = sp.hess_diag(xt, c1, c2, 4, c3=C3).cpu().numpy().astype(np.float64)
        P = np.zeros((len(V), 3, 3))
        P[:, [0, 1, 2], [0, 1, 2]] = planes[0]
        P[:, 1, 2] = P[:, 2, 1] = planes[1][:, 0]
        P[:, 0, 2] = P[:, 2, 0] = planes[1][:, 1]
        P[:, 0, 1] = P[:, 1, 0] = planes[1][:, 2]
        for S in classes[:3]:
            S = S[np.isin(S, np.unique(T))]
            for a in range(3):
                v = np.zeros((len(V), 3), np.float32)
                v[S, a] = 1.0
                hv, _ = sp.hvp(xt, torch.from_numpy(v).cuda(), c1, c2, 4, c3=C3)
                hv = hv.cpu().numpy().astype(np.float64)
                err = np.abs(hv[S] - P[S, :, a]).max(axis=1)
                assert (err <= 2 * KAPPA * U * A[S]).all(), (case, a, (err / (U * A[S])).max())


@pytest.mark.gpu
@pytest.mark.parametrize("mesh,kw", plan_shape_cases())
def test_hess_diag_plan_shapes(ext, mesh, kw):
    """The diagonal blocks per row on the plans only these meshes produce (assert_plan_shape): the pole's row 0 sums its
    988 weights in one ring-wrapping row block and its 1972 tets' blocks."""
    V, T, *_ = _refs(mesh)
    sp = _handle(ext, V, T, enable_amips=True, **kw)
    check_handle_plan_shape(mesh, sp, kw, enable_amips=True)
    _check_against_fp64(sp, mesh, str(kw))


def _call(sp, x, terms, out, stream, gradH=1.0, gradH_dev=None):
    from tssplat_b200 import _capi
    return _capi.lib.tsb_hess_diag(sp._h, x.data_ptr() if x is not None else None, C.byref(terms) if terms is not None else None,
                                   gradH, gradH_dev, out.data_ptr() if out is not None else None, stream)


@pytest.mark.gpu
def test_gradH_scaling(ext):
    """gradH and *gradH_dev multiply every entry: a power of two scales each bitwise on a deterministic handle."""
    torch = _torch()
    V, T, _, _, cases = _refs("shuffled")
    sp = _handle(ext, V, T, enable_amips=True, deterministic=True)
    x = torch.from_numpy(cases["inverted_o2"][0]).cuda()
    d1 = sp.hess_diag(x, 2e-3, 0.8, 2, c3=C3)
    d2 = sp.hess_diag(x, 2e-3, 0.8, 2, c3=C3, gradH=2.0)
    d3 = sp.hess_diag(x, 2e-3, 0.8, 2, c3=C3, gradH=torch.tensor(2.0, device="cuda"))
    d4 = sp.hess_diag(x, 2e-3, 0.8, 2, c3=C3, gradH=0.7)
    torch.cuda.synchronize()
    assert torch.equal(d2, 2 * d1) and torch.equal(d3, d2)
    assert float((d4 - 0.7 * d1).abs().max()) <= 1e-6 * float(d1.abs().max())
    # the module-level form, and the out= argument
    out = torch.full_like(d1, float("nan"))
    assert sp.hess_diag(x, 2e-3, 0.8, 2, c3=C3, out=out) is out and torch.equal(out, d1)
    ext_default = _handle(ext, V, T)
    dm = ext.hess_diag(x, ext_default, 2e-3, 0.8, 2)
    d0 = sp.hess_diag(x, 2e-3, 0.8, 2)
    orph = torch.ones(len(V), dtype=torch.bool)
    orph[torch.from_numpy(np.unique(T)).long()] = False
    assert not dm[:, orph.cuda()].any()
    assert float((dm - d0).abs().max()) <= 1e-6 * float(d0.abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(force_global=True, warps_per_cta=8)], ids=["staged", "global-w8"])
def test_deterministic_bitwise(ext, kw):
    """Deterministic handles: the same bits across launches, streams, graph replays and handles; rows no active tet
    touches are bitwise those of a default handle."""
    torch = _torch()
    from tssplat_b200 import _capi
    V, T, _, _, cases = _refs("pack64x4096")
    x = torch.from_numpy(cases["inverted_o2"][0]).cuda()
    det = _handle(ext, V, T, enable_amips=True, deterministic=True, **kw)
    det2 = _handle(ext, V, T, enable_amips=True, deterministic=True, **kw)
    c1, c2 = 2e-3, 0.8
    d0 = det.hess_diag(x, c1, c2, 2, c3=C3, gradH=GH)
    for _ in range(2):
        assert torch.equal(d0, det.hess_diag(x, c1, c2, 2, c3=C3, gradH=GH))
    assert torch.equal(d0, det2.hess_diag(x, c1, c2, 2, c3=C3, gradH=GH))
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=C3)
    s = torch.cuda.Stream()
    out = torch.empty_like(d0)
    with torch.cuda.stream(s):
        assert _call(det, x, terms, out, s.cuda_stream, gradH=GH) == 0
    s.synchronize()
    assert torch.equal(out, d0)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        assert _call(det, x, terms, out, s.cuda_stream, gradH=GH) == 0
    for _ in range(3):
        out.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, d0)
    # rows without active tets (c3 = 0: only the inverted spheres' vertices have tet blocks)
    plain = _handle(ext, V, T, **kw)
    dd = det.hess_diag(x, c1, c2, 2, gradH=GH)
    dp = plain.hess_diag(x, c1, c2, 2, gradH=GH)
    Tn = np.asarray(T, np.int64)
    xn = cases["inverted_o2"][0].astype(np.float64)
    e = lambda k: xn[Tn[:, k]] - xn[Tn[:, 0]]
    inv = (e(1) * np.cross(e(2), e(3))).sum(axis=1) < 0
    touched = np.zeros(len(V), bool)
    touched[np.unique(Tn[inv])] = True
    quiet = torch.from_numpy(~touched).cuda()
    assert touched.any() and (~touched).any()
    assert torch.equal(dd[:, quiet], dp[:, quiet])
    assert float((dd - dp).abs().max()) <= 1e-6 * float(dp.abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(force_global=True), dict(deterministic=True),
                                dict(deterministic=True, force_global=True, warps_per_cta=8)],
                         ids=["staged", "global", "det", "det-global-w8"])
def test_chaining_leaves_other_calls_unchanged(ext, kw):
    """energy_grad_ex, hess_diag, energy_grad_ex, hvp_ex on one stream give what a handle that never ran hess_diag
    gives: bitwise, on an input where no tet adds with atomics on a default handle (c3 = 0, no inverted tet) and with
    every term on a deterministic handle."""
    torch = _torch()
    V, T, _, _, cases = _refs("pack64x4096")
    det = bool(kw.get("deterministic"))
    x_np = cases["inverted_o2" if det else "benign_o2"][0]
    c3 = C3 if det else 0.0
    x = torch.from_numpy(x_np).cuda()
    x2 = torch.from_numpy((x_np * np.float32(1.001)).astype(np.float32)).cuda()
    w = torch.from_numpy(np.random.default_rng(2).normal(size=x_np.shape).astype(np.float32)).cuda()
    a, b = _handle(ext, V, T, enable_amips=True, **kw), _handle(ext, V, T, enable_amips=True, **kw)
    c1, c2 = 2e-3, 0.8
    res = []
    for h, run_diag in ((a, True), (b, False)):
        e1, g1 = h.energy_grad(x, c1, c2, 2, c3=c3)
        e1 = e1.clone()
        if run_diag:
            h.hess_diag(x, c1, c2, 2, c3=c3)
        e2, g2 = h.energy_grad(x2, c1, c2, 2, c3=c3)
        e2 = e2.clone()
        hv, cv = h.hvp(x2, w, c1, c2, 2, want_curv=True, c3=c3)
        res.append((e1, g1, e2, g2, hv, cv))
    torch.cuda.synchronize()
    for p, q in zip(*res):
        assert torch.equal(p, q)


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["plain", "amips"])
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
@pytest.mark.parametrize("nw", [16, 8], ids=["w16", "w8"])
def test_handle_info_unchanged(ext, amips, det, nw):
    """The DIAG instantiations add no plan data, shared memory, grid or device memory: the values pinned before the
    Hessian diagonal existed, also after a call."""
    torch = _torch()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("the pinned values are those of a 132-SM H100")
    from test_hvp_amips import _INFO_PINS
    V, T, _, _, cases = _refs("pack64x4096")
    sp = _handle(ext, V, T, enable_amips=amips, deterministic=det, warps_per_cta=nw)
    info0 = dict(sp.info)
    assert (info0["grid"], info0["smem_bytes"], info0["device_bytes"]) == _INFO_PINS[(amips, det, nw)]
    sp.hess_diag(torch.from_numpy(cases["benign_o2"][0]).cuda(), 1.0, 1.0, 2, c3=C3 if amips else 0.0)
    torch.cuda.synchronize()
    from tssplat_b200 import _capi
    info = _capi.tsb_info_t()
    _capi.check(_capi.lib.tsb_get_info(sp._h, C.byref(info)), sp._h)
    assert {k: getattr(info, k) for k, _ in _capi.tsb_info_t._fields_} == info0


@pytest.mark.gpu
def test_bad_arguments(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    V, T, _, _, cases = _refs("shuffled")
    plain, am = _handle(ext, V, T), _handle(ext, V, T, enable_amips=True)
    x = torch.from_numpy(cases["benign_o2"][0]).cuda()
    out = torch.full((2, len(V), 3), float("nan"), device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    E = _capi.TSB_E_INVALID
    good = _capi.tsb_terms_t(c1=1.0, c2=1.0, order=2, c3=0.5)
    assert _call(plain, x, good, out, st) == E                                     # c3 != 0 without enable_amips
    assert "enable_amips" in _capi.last_error(plain._h)
    with pytest.raises(RuntimeError, match="enable_amips"):
        plain.hess_diag(x, 1.0, 1.0, 2, c3=0.5)
    assert _call(am, x, None, out, st) == E
    assert _call(am, None, good, out, st) == E
    assert _call(am, x, good, None, st) == E
    assert _call(am, x, _capi.tsb_terms_t(c1=1.0, c2=1.0, order=3, c3=0.5), out, st) == E
    assert _capi.lib.tsb_hess_diag(None, x.data_ptr(), C.byref(good), 1.0, None, out.data_ptr(), st) == E
    torch.cuda.synchronize()
    assert torch.isnan(out).all()                                                   # nothing was launched
    with pytest.raises(RuntimeError):
        am.hess_diag(x, 1.0, 1.0, 2, out=torch.empty((len(V), 3), device="cuda"))


@pytest.mark.gpu
def test_module_hess_diag(ext):
    """SmoothnessBarrierEnergy.hess_diag uses the scheduler's coefficients, order_at(it) and amips_coeff."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    V, T, _, _, cases = _refs("shuffled")
    E = SmoothnessBarrierEnergy(V, T.reshape(-1, 4), dict(smooth_eng_coeff=2e-3, barrier_coeff=0.8, increase_order_iter=100,
                                                          deterministic=True, amips_coeff=C3))
    x = torch.from_numpy(cases["inverted_o2"][0]).cuda().requires_grad_(True)
    for it in (10, 500):
        c1, c2 = E.coeff_scheduler(it)
        assert torch.equal(E.hess_diag(x, it), E.tet_sp.hess_diag(x.detach(), c1, c2, E.order_at(it), c3=C3))


@pytest.mark.gpu
def test_block_jacobi_pcg_end_to_end(ext):
    """On make_pack(3, 512, seed=4) near rest, CG with the block-Jacobi preconditioner of hess_diag reaches
    |r| <= 1e-3 |b| in fewer Hessian-vector products than plain CG, and its step decreases the energy."""
    torch = _torch()
    from tssplat_b200.newton import block_jacobi, pcg
    pk = make_pack(3, 512, seed=4)
    sp = _handle(ext, pk.verts, pk.tets)
    x = torch.from_numpy(perturb(pk, sigma_rel=0.02, seed=1)).cuda()
    c1, c2 = 2e-4 / 3, 2e-4
    e0, g = sp.energy_grad(x, c1, c2, 2)
    e0 = float(e0[0])
    b = -g
    hvp = lambda p: sp.hvp(x, p, c1, c2, 2)[0]
    P = block_jacobi(sp.hess_diag(x, c1, c2, 2))
    plain = pcg(hvp, b, None, max_iter=500, rtol=1e-3)
    pre = pcg(hvp, b, P, max_iter=500, rtol=1e-3)
    print(f"CG to 1e-3: {plain.n_hvp} products unpreconditioned, {pre.n_hvp} with block Jacobi")
    assert plain.converged and pre.converged and not pre.negative_curvature
    assert pre.n_hvp < plain.n_hvp
    e1, _ = sp.energy_grad(x + pre.x, c1, c2, 2, want_grad=False)
    assert float(e1[0]) < e0
