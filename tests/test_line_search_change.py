"""The line search's energy changes (tsb_line_search) against fp64 to the size of the change, term by term, per sphere
and in total.

Every device Newton rule accepts or rejects a step on these changes (the Armijo test, the gain ratio), so they must be
accurate relative to their own size, which can be far below the energy: at small alpha, near a minimum, or when a sphere
has moved far from rest.  The kernel forms each change without subtracting two energies (DESIGN.md section 5, "Line
search"); this file holds it to that.

CPU: change_ref, the changes in the kernel's cancellation-free forms evaluated in fp64 on the exact fp32 inputs (x, d,
the plan's fp32 1/det(Dm), rest inverses and operator weights), checked against mpmath at 50 digits (naive differences)
and against the oracle's gradient and Hessian-vector product in the small-alpha limit; rounding scales A (first-order
propagation of fp32 rounding through the kernel's formulas, on absolute values); reenact_fp32, the kernel's per-tet
LINE branch and row end restated in fp32, which calibrates KAPPA; four regressions (plain differences per tet and per
row, a dropped reference shift, a cubic built from absolute corner values of d) that pass the old energy-relative
bound and fail this one by more than 100x.  GPU: every handle kind at orders 2 and 4, AMIPS off and on, alpha = 2^-k
(k = 0..23) and 0.3 * 2^-k, on benign, inverted, near-converged, moved, translated and scaling inputs and on single
tets at J near 0; known answers for translations; the sign of the Armijo margin."""
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sps

from _helpers import check_handle_plan_shape, plan_shape_cases, rigid_motion
from test_line_search import REL, components, line_terms, make_oracle
from test_psd_edges import single_tet_mesh
from tssplat_b200.mesh import make_pack, perturb

U = 2.0 ** -24                  # fp32 unit roundoff
# |change_gpu - change_64| <= KAPPA u A + u |change_64| per term, per sphere and in total (test_kappa_calibration: the
# fp32 restatement must stay within KAPPA / 4 on random inputs and on every edge family)
KAPPA = 16
C1, C2, C3 = 2e-3, 0.8, 1e-4
SIGMA = 1e-4                    # Armijo constant of the agreement check
LADDER = [2.0 ** -k for k in range(24)]
POINT3 = [0.3 * 2.0 ** -k for k in (0, 8, 16)]
LAUNCHES = [LADDER[0:8], LADDER[8:16], LADDER[16:24], POINT3]      # TSB_LINE_MAX_ALPHA = 8 step sizes per launch
TERMS = ("smooth", "barrier", "amips")

f32, f64 = np.float32, np.float64


# ---------------------------------------------------------------------------------------------------------------------
# the plan's fp32 data and the fp64 reference


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def _dot(a, b):
    return (a * b).sum(axis=-1)


class Geo:
    """A mesh as the kernel sees it: fp32 rest positions, 1/det(Dm) rounded to fp32 (tsb_plan.cpp emit_tc), the rest
    inverse B rounded to fp32 (the AMIPS blocks), the operator's off-diagonal weights rounded to fp32 with the diagonal
    their negated row sum (the row pass forms sum_j w_ij (u_j - u_i)), and each component's reference vertex, its
    lowest vertex id.  exact=True keeps all of them in fp64 (the oracle's operators: the Taylor checks)."""

    def __init__(self, V, T, exact=False):
        rnd = (lambda a: a) if exact else (lambda a: np.asarray(a, f32).astype(f64))
        self.V32 = np.ascontiguousarray(V, f32).reshape(-1, 3)
        self.X = self.V32.astype(f64)
        self.T = np.asarray(T, np.int64).reshape(-1, 4)
        self.n, self.nt = len(self.X), len(self.T)
        Dm = self.X[self.T[:, 1:]] - self.X[self.T[:, :1]]                    # [t, k, r]: edge k
        det = _dot(Dm[:, 0], _cross(Dm[:, 1], Dm[:, 2]))
        self.idet = rnd(1.0 / det)
        self.B = rnd(np.linalg.inv(Dm.transpose(0, 2, 1)))                   # B = Dm^-1, Dm columns = edges
        self.orc = orc = make_oracle(self.V32, self.T)
        m = orc.M[0::3, 0::3].tocoo()                                        # M = m (x) I_3
        off = (m.row != m.col) & (m.data != 0)
        self.W = sps.csr_matrix((rnd(m.data[off]), (m.row[off], m.col[off])), shape=(self.n, self.n))
        self.W.sort_indices()
        self.wsum = np.asarray(self.W.sum(axis=1)).ravel()
        self.vlab, self.tlab, self.S = components(self.V32, self.T)
        used = self.vlab >= 0
        self.ref = np.array([np.flatnonzero(self.vlab == c)[0] for c in range(self.S)])
        self.rv = np.where(used, self.ref[np.maximum(self.vlab, 0)], np.arange(self.n))
        self.used = used
        self.h = float(np.linalg.norm(Dm, axis=2).mean())


def _sphere_sum(lab, S, v):
    m = lab >= 0
    return np.bincount(lab[m], weights=v[m], minlength=S)


class Prep:
    """Everything of change_ref that does not depend on alpha, for one (x, d) on one Geo."""

    def __init__(self, g, x32, d32):
        x32 = np.ascontiguousarray(x32, f32).reshape(-1, 3)
        d32 = np.ascontiguousarray(d32, f32).reshape(-1, 3)
        self.g, self.x32, self.d32 = g, x32, d32
        x, d = x32.astype(f64), d32.astype(f64)
        rv = g.rv
        # rows: u_i - c with c = fp32(x_r - X_r) (rel_u), d_i - d_r (the staged direction), M d = sum_j w_ij (d_j - d_i)
        c = (x32[rv] - g.V32[rv]).astype(f64)                                # fp32 subtraction, as the kernel
        self.uc = (x - g.X) - c
        self.dr = d - d[rv]
        Md = g.W @ self.dr - g.wsum[:, None] * self.dr
        self.row1 = _dot(self.uc, Md)                                         # alpha u^T M d, per row
        self.row2 = 0.5 * _dot(self.dr, Md)                                   # 1/2 alpha^2 d^T M d, per row
        # scale: S_i = sum_j |w_ij| (|d_j - d_i| + |w_j| + |w_i|) per coordinate (w: the staged d - d_r, whose rounding
        # enters every difference), A_s = alpha sum |u_i - c| S_i + 1/2 alpha^2 sum (|d_i - d_r| + D_c) S_i, D_c the
        # largest |d_j - d_r| of the component (the row end subtracts the staged value at staging position 0)
        Wc = g.W.tocoo()
        ad = np.abs(self.dr)
        Srow = np.zeros((g.n, 3))
        for r in range(3):
            Srow[:, r] = np.bincount(Wc.row, weights=np.abs(Wc.data) * (np.abs(self.dr[Wc.col, r] - self.dr[Wc.row, r])
                                                                       + ad[Wc.col, r] + ad[Wc.row, r]), minlength=g.n)
        Dc = np.zeros((g.S + 1, 3))
        for r in range(3):
            np.maximum.at(Dc[:, r], np.where(g.used, g.vlab, g.S), ad[:, r])
        Dv = Dc[np.where(g.used, g.vlab, g.S)]
        self.arow1 = _dot(np.abs(self.uc), Srow)
        self.arow2 = 0.5 * _dot(ad + Dv, Srow)
        # tets: edges of x and of d (exact differences of the fp32 inputs), the cubic J(alpha) = J0 + J1 a + J2 a^2 + J3 a^3
        T = g.T
        e = x[T[:, 1:]] - x[T[:, :1]]
        f = d[T[:, 1:]] - d[T[:, :1]]
        w = np.abs(self.dr)                                                   # |staged d - d_r|
        c1, c2, c3 = _cross(e[:, 1], e[:, 2]), _cross(e[:, 2], e[:, 0]), _cross(e[:, 0], e[:, 1])
        g1 = _cross(f[:, 1], f[:, 2])
        idet = g.idet
        self.J0 = _dot(e[:, 0], c1) * idet
        self.J1 = (_dot(f[:, 0], c1) + _dot(f[:, 1], c2) + _dot(f[:, 2], c3)) * idet
        self.J2 = (_dot(e[:, 0], g1) + _dot(e[:, 1], _cross(f[:, 2], f[:, 0])) + _dot(e[:, 2], _cross(f[:, 0], f[:, 1]))) * idet
        self.J3 = _dot(f[:, 0], g1) * idet
        ne = np.linalg.norm(e, axis=2)
        nf = np.linalg.norm(f, axis=2) + np.linalg.norm(w[T[:, 1:]], axis=2) + np.linalg.norm(w[T[:, :1]], axis=2)
        ai = np.abs(idet)
        self.Jh0 = ai * ne[:, 0] * ne[:, 1] * ne[:, 2]
        self.Jh1 = ai * (nf[:, 0] * ne[:, 1] * ne[:, 2] + ne[:, 0] * nf[:, 1] * ne[:, 2] + ne[:, 0] * ne[:, 1] * nf[:, 2])
        self.Jh2 = ai * (ne[:, 0] * nf[:, 1] * nf[:, 2] + nf[:, 0] * ne[:, 1] * nf[:, 2] + nf[:, 0] * nf[:, 1] * ne[:, 2])
        self.Jh3 = ai * nf[:, 0] * nf[:, 1] * nf[:, 2]
        # AMIPS: F = E B, dF = f B (E, f with the edges as columns); I1(alpha) = tr + alpha (2 fdf + alpha dd)
        F = np.einsum("tkr,tkc->trc", e, g.B)
        D = np.einsum("tkr,tkc->trc", f, g.B)
        Fa = np.einsum("tkr,tkc->trc", np.abs(e), np.abs(g.B))
        Da = np.einsum("tk,tkc->tc", nf, np.abs(g.B))[:, None, :]         # |f_k| per row, as a bound
        self.tr, self.fdf, self.dd = (F * F).sum((1, 2)), (F * D).sum((1, 2)), (D * D).sum((1, 2))
        self.Ia = (Fa * Fa).sum((1, 2))
        self.fda = (Fa * Da).sum((1, 2))
        self.dda = 3 * (Da * Da).sum((1, 2))


def tet_terms(p, a, order, kappa=KAPPA, amips=True):
    """Per tet at step alpha = a: (db, da) in the kernel's forms in fp64, their rounding scales (Ab, Aa), the barrier's
    allowance for tets whose sign fp32 may decide either way, and the tets whose AMIPS activity fp32 may decide either
    way (not comparable: psi has a pole at J = 0)."""
    J0, Jh0 = p.J0, p.Jh0
    dJ = a * (p.J1 + a * (p.J2 + a * p.J3))
    Ja = J0 + dJ
    Jhat = a * (p.Jh1 + a * (p.Jh2 + a * p.Jh3))
    Jt1 = Jh0 + Jhat
    m0, m = np.maximum(-J0, 0.0), np.maximum(-Ja, 0.0)
    both = (J0 < 0) & (Ja < 0)
    if order == 2:
        db = np.where(both, -dJ * (m + m0), m * m - m0 * m0)
    else:
        db = np.where(both, -dJ * (m + m0) * (m * m + m0 * m0), m ** 4 - m0 ** 4)
    cross = (J0 < 0) != (Ja < 0)
    Ab = np.where((J0 < 0) | (Ja < 0), order * (np.maximum(m, m0) + Jt1) ** (order - 1) * (Jhat + np.where(cross, Jh0, 0.0)), 0.0)
    # J within kappa u of its scale at an end: fp32 may put it on either side of 0, where that end's barrier is at most
    # (|J| + kappa u Jhat)^p
    amb0, amb1 = np.abs(J0) <= kappa * U * Jh0, np.abs(Ja) <= kappa * U * Jt1
    amb = amb0 | amb1
    allow_b = np.where(amb, np.abs(db) + amb0 * (np.abs(J0) + kappa * U * Jh0) ** order
                       + amb1 * (np.abs(Ja) + kappa * U * Jt1) ** order, 0.0)
    if not amips:
        return SimpleNamespace(db=db, Ab=Ab, allow_b=allow_b, J=Ja)
    # AMIPS
    act0, act1 = J0 > 0, Ja > 0
    with np.errstate(all="ignore"):
        r0 = np.cbrt(np.where(act0, J0, 1.0))
        r = np.cbrt(np.where(act1, Ja, 1.0))
        q = 1.0 / (3.0 * r * r)
        q0 = 1.0 / (3.0 * r0 * r0)
        dI = a * (2.0 * p.fdf + a * p.dd)
        dIa = a * (2.0 * p.fda + a * p.dda)
        k2 = (r0 + r) * q / (r0 * r0 * (r * (r + r0) + r0 * r0))
        da_both = dI * q - p.tr * dJ * k2
        Aa_both = dIa * q * (1 + Jt1 / Ja) + p.Ia * (Jhat + np.abs(dJ) * (1 + Jh0 / J0 + Jt1 / Ja)) * k2
        da = np.where(act0 & act1, da_both, np.where(act1, (p.tr + dI) * q - 1.0, np.where(act0, 1.0 - p.tr * q0, 0.0)))
        Aa = np.where(act0 & act1, Aa_both, np.where(act1, (p.Ia + dIa) * q * (1 + Jt1 / Ja) + 1.0,
                                                     np.where(act0, p.Ia * q0 * (1 + Jh0 / J0) + 1.0, 0.0)))
    return SimpleNamespace(db=db, da=da, Ab=Ab, Aa=Aa, allow_b=allow_b, amb_a=amb, J=Ja)


class Ref:
    """change_ref of one (x, d) on one Geo at the fp32 step sizes alphas, summed per sphere: arrays [K, S] of the three
    terms (smooth, barrier order 2 and 4, AMIPS), their scales and allowances, and [K, S] masks of the spheres whose AMIPS
    change is not comparable at alpha_k."""

    def __init__(self, g, x32, d32, alphas, prep=None):
        p = prep if prep is not None else Prep(g, x32, d32)
        self.p = p
        al = np.asarray(np.asarray(alphas, f32), f64)
        self.alphas = al
        S = g.S
        rs1, rs2 = _sphere_sum(g.vlab, S, p.row1), _sphere_sum(g.vlab, S, p.row2)
        ra1, ra2 = _sphere_sum(g.vlab, S, p.arow1), _sphere_sum(g.vlab, S, p.arow2)
        self.ds = np.array([a * rs1 + a * a * rs2 for a in al])
        self.As = np.array([a * ra1 + a * a * ra2 for a in al])
        self.db, self.Ab, self.allow_b = {2: [], 4: []}, {2: [], 4: []}, {2: [], 4: []}
        self.da, self.Aa, self.amb_a = [], [], []
        for a in al:
            for order in (4, 2):
                t = tet_terms(p, a, order, amips=order == 2)
                self.db[order].append(_sphere_sum(g.tlab, S, t.db))
                self.Ab[order].append(_sphere_sum(g.tlab, S, t.Ab))
                self.allow_b[order].append(_sphere_sum(g.tlab, S, t.allow_b))
            self.da.append(_sphere_sum(g.tlab, S, t.da))
            self.Aa.append(_sphere_sum(g.tlab, S, t.Aa))
            self.amb_a.append(_sphere_sum(g.tlab, S, t.amb_a.astype(f64)) > 0)
        for k in ("db", "Ab", "allow_b"):
            setattr(self, k, {o: np.array(v) for o, v in getattr(self, k).items()})
        self.da, self.Aa, self.amb_a = np.array(self.da), np.array(self.Aa), np.array(self.amb_a)

    def term(self, j, order, c3):
        """(value, scale, allowance) [K, S] of column j (1 smooth, 2 barrier, 3 AMIPS) as the launch computes it."""
        z = np.zeros_like(self.ds)
        if j == 1:
            return self.ds, self.As, z
        if j == 2:
            return self.db[order], self.Ab[order], self.allow_b[order]
        return (self.da, self.Aa, z) if c3 else (z, z, z)


def ratio(err, val, A, allow=0.0):
    """How much of the bound KAPPA u A + u |val| + allow the error uses, in units of u A: (|err| - u |val| - allow) / (u
    A), 0 when within the output rounding; inf when A = 0 and the error is not."""
    ex = np.maximum(np.abs(err) - U * np.abs(val) - allow, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(ex == 0, 0.0, ex / (U * A))


# ---------------------------------------------------------------------------------------------------------------------
# the kernel's LINE branch restated in fp32


def _fma(a, b, c):
    """fmaf approximated: one fp64 multiply-add (the product of two floats is exact in fp64) rounded to fp32."""
    return (np.asarray(a, f64) * np.asarray(b, f64) + np.asarray(c, f64)).astype(f32)


def _rel_u(x, X, c):
    s = x - X
    bb = s - x
    e = (x - (s - bb)) + (-X - bb)
    return (s - c) + e


def reenact_fp32(g, x32, d32, alphas, order, mutation=None):
    """The LINE per-tet branch (barrier and AMIPS changes per tet) and row end (alpha u^T M d + 1/2 alpha^2 d^T M d per
    row) of energy_grad_kernel in fp32 numpy, operation for operation as written in the source.  fmaf is emulated by
    _fma and cbrtf by numpy's fp32 cbrt: both approximations (rounding may differ in the last place, and nvcc may
    contract other products into FMAs).  The row pass accumulates each row's entries in one fp32 chain (the kernel: two
    interleaved chains, added at the end).

    mutation: the regressions of test_regressions_fail_the_new_bound -- "plain_tet" (m(alpha)^p - m0^p and psi(alpha) -
    psi(0) in fp32), "plain_smooth" (1/2 u(alpha)^T M u(alpha) - 1/2 u^T M u per row in fp32), "no_shift" (u_i = x_i -
    X_i without the component's c), "corner_dF" (J1, J2, J3 from dF = sum_k d_k a_k^T over the absolute corner values
    of d, as G d forms it, instead of the staged edges).
    Returns per-row ds [K, n] and per-tet db, da [K, T] (fp64 of the fp32 values)."""
    T = g.T
    x32 = np.ascontiguousarray(x32, f32).reshape(-1, 3)
    d32 = np.ascontiguousarray(d32, f32).reshape(-1, 3)
    X32 = g.V32
    rv = g.rv
    w = d32 - d32[rv]                                                        # staged d - d_r
    idet = g.idet.astype(f32)
    al32 = np.asarray(alphas, f32)
    # ---- row end
    Wc = g.W
    n = g.n
    ax = np.zeros((n, 3), f32)
    lens = np.diff(Wc.indptr)
    for s in range(int(lens.max()) if len(lens) else 0):
        rows = np.flatnonzero(lens > s)
        idx = Wc.indptr[rows] + s
        wij = Wc.data[idx].astype(f32)[:, None]
        ax[rows] = _fma(wij, w[Wc.indices[idx]] - w[rows], ax[rows])
    lc = (x32[rv] - X32[rv])
    ui = w
    des = _fma(ui[:, 0], ax[:, 0], _fma(ui[:, 1], ax[:, 1], ui[:, 2] * ax[:, 2])).astype(f64)
    if mutation == "no_shift":
        uu = x32 - X32
    else:
        uu = _rel_u(x32, X32, lc)
    deb = _fma(uu[:, 0], ax[:, 0], _fma(uu[:, 1], ax[:, 1], uu[:, 2] * ax[:, 2])).astype(f64)
    ds = []
    for a in al32.astype(f64):
        ds.append(a * deb + 0.5 * (a * a) * des)
    if mutation == "plain_smooth":
        # 1/2 u(alpha)_i . (M u(alpha))_i - 1/2 u_i . (M u)_i with u(alpha) = fp32(u + alpha d), u = rel_u
        def half_uMu(v):
            acc = np.zeros((n, 3), f32)
            for s in range(int(lens.max())):
                rows = np.flatnonzero(lens > s)
                idx = Wc.indptr[rows] + s
                acc[rows] = _fma(Wc.data[idx].astype(f32)[:, None], v[Wc.indices[idx]] - v[rows], acc[rows])
            return f32(0.5) * _fma(v[:, 0], acc[:, 0], _fma(v[:, 1], acc[:, 1], v[:, 2] * acc[:, 2]))
        e0 = half_uMu(uu)
        ds = [(half_uMu((uu + a * w).astype(f32)) - e0).astype(f64) for a in al32]
    # ---- per tet
    xv = x32[T]
    e1, e2, e3 = (xv[:, k] - xv[:, 0] for k in (1, 2, 3))
    c1 = np.stack([e2[:, 1] * e3[:, 2] - e2[:, 2] * e3[:, 1], e2[:, 2] * e3[:, 0] - e2[:, 0] * e3[:, 2],
                   e2[:, 0] * e3[:, 1] - e2[:, 1] * e3[:, 0]], 1)
    J = (e1[:, 0] * c1[:, 0] + e1[:, 1] * c1[:, 1] + e1[:, 2] * c1[:, 2]) * idet
    wv = w[T]
    f1, f2, f3 = (wv[:, k] - wv[:, 0] for k in (1, 2, 3))
    cr = lambda a, b: np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                                a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    dt = lambda a, b: a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1] + a[:, 2] * b[:, 2]
    g1 = cr(f2, f3)
    if mutation == "corner_dF":
        B = g.B.astype(f32)
        dv = d32[T]
        a0 = -(B[:, 0] + B[:, 1] + B[:, 2])
        Fm = (e1[:, :, None] * B[:, 0, None, :] + e2[:, :, None] * B[:, 1, None, :]) + e3[:, :, None] * B[:, 2, None, :]
        dF = ((dv[:, 0, :, None] * a0[:, None, :] + dv[:, 1, :, None] * B[:, 0, None, :])
              + dv[:, 2, :, None] * B[:, 1, None, :]) + dv[:, 3, :, None] * B[:, 2, None, :]
        cof = lambda A, C: np.stack([cr(A[:, 1], C[:, 2]), cr(A[:, 2], C[:, 0]), cr(A[:, 0], C[:, 1])], 1)  # rows
        # J(F + a dF) with rows r: J1 = sum_r dF_r . (F_{r+1} x F_{r+2}), J2 = sum_r F_r . (dF_{r+1} x dF_{r+2}), J3 = det dF
        cF, cD = cof(Fm, Fm), cof(dF, dF)
        J1 = (dF * cF).sum((1, 2), dtype=f32)
        J2 = (Fm * cD).sum((1, 2), dtype=f32)
        J3 = dt(dF[:, 0], cr(dF[:, 1], dF[:, 2]))
    else:
        J1 = (dt(f1, c1) + f2[:, 0] * (e3[:, 1] * e1[:, 2] - e3[:, 2] * e1[:, 1]) + f2[:, 1] * (e3[:, 2] * e1[:, 0] - e3[:, 0] * e1[:, 2])
              + f2[:, 2] * (e3[:, 0] * e1[:, 1] - e3[:, 1] * e1[:, 0]) + f3[:, 0] * (e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1])
              + f3[:, 1] * (e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]) + f3[:, 2] * (e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0])) * idet
        J2 = (dt(e1, g1) + e2[:, 0] * (f3[:, 1] * f1[:, 2] - f3[:, 2] * f1[:, 1]) + e2[:, 1] * (f3[:, 2] * f1[:, 0] - f3[:, 0] * f1[:, 2])
              + e2[:, 2] * (f3[:, 0] * f1[:, 1] - f3[:, 1] * f1[:, 0]) + e3[:, 0] * (f1[:, 1] * f2[:, 2] - f1[:, 2] * f2[:, 1])
              + e3[:, 1] * (f1[:, 2] * f2[:, 0] - f1[:, 0] * f2[:, 2]) + e3[:, 2] * (f1[:, 0] * f2[:, 1] - f1[:, 1] * f2[:, 0])) * idet
        J3 = dt(f1, g1) * idet
    B = g.B.astype(f32)
    tr = np.zeros(len(T), f32)
    fdf, dd = tr.copy(), tr.copy()
    for c in range(3):
        Fc = [e1[:, r] * B[:, 0, c] + e2[:, r] * B[:, 1, c] + e3[:, r] * B[:, 2, c] for r in range(3)]
        Dc = [f1[:, r] * B[:, 0, c] + f2[:, r] * B[:, 1, c] + f3[:, r] * B[:, 2, c] for r in range(3)]
        tr = _fma(Fc[0], Fc[0], _fma(Fc[1], Fc[1], _fma(Fc[2], Fc[2], tr)))
        fdf = _fma(Fc[0], Dc[0], _fma(Fc[1], Dc[1], _fma(Fc[2], Dc[2], fdf)))
        dd = _fma(Dc[0], Dc[0], _fma(Dc[1], Dc[1], _fma(Dc[2], Dc[2], dd)))
    with np.errstate(all="ignore"):
        r0 = np.where(J > 0, np.cbrt(J), f32(0))
        dbs, das = [], []
        for al in al32:
            dJ = al * _fma(al, _fma(al, J3, J2), J1)
            Ja = J + dJ
            m0, m = np.maximum(-J, f32(0)), np.maximum(-Ja, f32(0))
            if mutation == "plain_tet":
                db = m * m - m0 * m0 if order == 2 else (m * m) * (m * m) - (m0 * m0) * (m0 * m0)
            else:
                qb = -dJ * (m + m0)
                both = qb if order == 2 else qb * _fma(m, m, m0 * m0)
                mm, mm0 = m * m, m0 * m0
                db = np.where((Ja < 0) & (J < 0), both, mm - mm0 if order == 2 else mm * mm - mm0 * mm0)
            dI = al * _fma(al, dd, f32(2) * fdf)
            r = np.cbrt(np.where(Ja > 0, Ja, f32(1)))
            r2 = r * r
            q = f32(1) / (f32(3) * r2)
            r02 = r0 * r0
            if mutation == "plain_tet":
                psi1 = (tr + dI) * q - f32(1)
                psi0 = tr / (f32(3) * r02) - f32(1)
                da = np.where(Ja > 0, np.where(J > 0, psi1 - psi0, psi1), np.where(J > 0, -psi0, f32(0)))
            else:
                da_both = dI * q - tr * dJ * (r0 + r) * q / (r02 * _fma(r, r + r0, r02))
                da = np.where(Ja > 0, np.where(J > 0, da_both, (tr + dI) * q - f32(1)),
                              np.where(J > 0, f32(1) - tr / (f32(3) * r02), f32(0)))
            dbs.append(db.astype(f64))
            das.append(da.astype(f64))
    return np.array(ds), np.array(dbs), np.array(das)


def per_tet_ratios(g, x32, d32, alphas, order, mutation=None):
    """Worst ratio per term of the fp32 restatement against change_ref, per row (smoothness) and per tet."""
    ds32, db32, da32 = reenact_fp32(g, x32, d32, alphas, order, mutation)
    p = Prep(g, x32, d32)
    al = np.asarray(np.asarray(alphas, f32), f64)
    out = dict(smooth=0.0, barrier=0.0, amips=0.0)
    for k, a in enumerate(al):
        ds64 = a * p.row1 + a * a * p.row2
        As = a * p.arow1 + a * a * p.arow2
        out["smooth"] = max(out["smooth"], ratio(ds32[k] - ds64, ds64, As)[g.used].max())
        t = tet_terms(p, a, order)
        out["barrier"] = max(out["barrier"], ratio(db32[k] - t.db, t.db, t.Ab, t.allow_b).max())
        ok = ~t.amb_a
        if ok.any():
            out["amips"] = max(out["amips"], ratio(da32[k][ok] - t.da[ok], t.da[ok], t.Aa[ok]).max())
    return out


# ---------------------------------------------------------------------------------------------------------------------
# inputs


def sphere_translations(g, scale, seed):
    """A different translation per sphere, of length `scale`, [n, 3] (0 on orphans)."""
    rng = np.random.default_rng(seed)
    t = rng.normal(size=(g.S, 3))
    t *= scale / np.linalg.norm(t, axis=1, keepdims=True)
    return np.where(g.used[:, None], t[np.maximum(g.vlab, 0)], 0.0)


def oracle_gradient(g, x32):
    """The fp64 oracle gradient of C1 smooth + C2 barrier (order 2) + C3 AMIPS at x, [n, 3]."""
    orc = g.orc
    x = np.asarray(x32, f32).astype(f64).reshape(-1, 3)
    gr = orc.backward(1.0, x, 0.0, C2, 2) + C1 * (orc.M @ (x - g.X).reshape(-1)).reshape(-1, 3)
    return gr + orc.amips_backward(1.0, x, C3)


def inputs(g, xb, xi, d, seed):
    """{name: (x32, d32)}: the benign and inverted inputs along d, near converged (rest + 1e-4 h, every J > 0) and the
    benign input along -g64, both moved by shift10 and rot1_far_pivot, d plus a per-sphere translation of 1e2 h and 1e4
    h, and the per-sphere scaling direction x - centroid."""
    rng = np.random.default_rng(seed)
    h = g.h
    xn = g.V32.copy()
    xn[g.used] += rng.normal(scale=1e-4 * h, size=(int(g.used.sum()), 3)).astype(f32)
    Jn = Prep(g, xn, np.zeros_like(xn)).J0
    assert (Jn > 0).all()
    gn, gb = -oracle_gradient(g, xn).astype(f32), -oracle_gradient(g, xb).astype(f32)
    cen = np.stack([_sphere_sum(g.vlab, g.S, xb[:, r].astype(f64)) for r in range(3)], 1)
    cnt = np.bincount(g.vlab[g.used], minlength=g.S)[:, None]
    scl = np.where(g.used[:, None], xb - (cen / cnt)[np.maximum(g.vlab, 0)], 0.0)
    out = {"benign": (xb, d), "inverted": (xi, d), "benign -g": (xb, gb), "near-converged -g": (xn, gn)}
    for name, shift, ang in (("shift10", 10.0, 0.0), ("rot1_far_pivot", 0.0, 1.0)):
        out[f"benign {name}"] = (rigid_motion(xb, shift, ang), d)
        out[f"near-converged {name}"] = (rigid_motion(xn, shift, ang), gn)
    for s in (1e2, 1e4):
        out[f"benign d+{s:.0e}h"] = (xb, (d + sphere_translations(g, s * h, seed + int(s))).astype(f32))
    out["benign scaling"] = (xb, scl.astype(f32))
    return {k: (np.ascontiguousarray(x, f32), np.ascontiguousarray(v, f32)) for k, (x, v) in out.items()}


J_FAMILY = [1e-2, 1e-4, 1e-6, 2.0 ** -20]


def _rot(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def single_tet_families():
    """(F per tet, label): J in {+-1e-2, +-1e-4, +-1e-6, +-2^-20} as diag(1, 1, J) and rotated, needles (singular values
    1, s, s with s = 1e-3 .. 1e-4, both signs), J = 0 exactly (a flat tet, a line, a point)."""
    Fs, lab = [], []
    for J in J_FAMILY:
        for sg in (1.0, -1.0):
            Fs.append(np.diag([1.0, 1.0, sg * J])); lab.append("J~0")
            Fs.append(_rot(len(Fs)) @ np.diag([1.0, 1.0, sg * J]) @ _rot(len(Fs) + 100)); lab.append("J~0")
    for s in (1e-3, 3e-4, 1e-4):
        for sg in (1.0, -1.0):
            Fs.append(_rot(len(Fs)) @ np.diag([1.0, s, sg * s]) @ _rot(len(Fs) + 100)); lab.append("needle")
    for F in (np.array([[1.0, 2.0, 3.0], [4.0, 5.0, 6.0], [0.0, 0.0, 0.0]]), np.array([[1.0, 1.0, 0.5], [0.0, 0.0, 0.0], [2.0, 2.0, 0.0]]),
              np.zeros((3, 3))):
        Fs.append(F); lab.append("J=0")
    for k in range(6):
        Fs.append(_rot(200 + k) @ np.diag([1.2, 0.9, 1.0 if k % 2 else -1.0]) @ _rot(300 + k)); lab.append("generic")
    return np.array(Fs), lab


def single_tet_case():
    """The single-tet mesh (each family on a unit right tet at the origin and on a generic rest tet far from it) and its
    directions: push (J(alpha) = J (1 - 3 alpha) on the unit tets: through zero at 1/3), pull (J (1 + 3 alpha)), and
    random corner moves of size 0.5 and 1e-3, and the first plus a translation of length 1e4 per tet."""
    Fs, lab = single_tet_families()
    V, T, x, B, F = single_tet_mesh(Fs, Fs)
    labels = [f"unit {s}" for s in lab] + [f"far {s}" for s in lab]
    nt = len(T)
    rng = np.random.default_rng(31)
    dirs = {}
    for name, k in (("push", -3.0), ("pull", 3.0)):
        # move corner 3 along F's third column (unit tets: x_3 = F e_3): J(alpha) = J (1 + k alpha); the far tets the same
        # relative to their edge 3
        dv = np.zeros((nt, 4, 3))
        dv[:, 3] = k * (x[:, 3].astype(f64) - x[:, 0].astype(f64))
        dirs[name] = dv
    for name, s in (("random", 0.5), ("small", 1e-3)):
        dirs[name] = rng.normal(scale=s, size=(nt, 4, 3))
    t = rng.normal(size=(nt, 1, 3))
    dirs["random+1e4"] = dirs["random"] + 1e4 * t / np.linalg.norm(t, axis=2, keepdims=True)
    return dict(V=V, T=T, x=x.reshape(-1, 3), labels=np.array(labels),
                dirs={k: np.asarray(v, f32).reshape(-1, 3) for k, v in dirs.items()})


# ---------------------------------------------------------------------------------------------------------------------
# CPU


@pytest.fixture(scope="module")
def small():
    pk = make_pack(3, 512, seed=4)
    g = Geo(pk.verts, pk.tets)
    rng = np.random.default_rng(5)
    xb = perturb(pk, sigma_rel=0.02, seed=1)
    xi = perturb(pk, sigma_rel=0.35, seed=2)
    d = rng.normal(scale=0.1 * g.h, size=pk.verts.shape).astype(f32)
    return SimpleNamespace(pk=pk, g=g, inputs=inputs(g, xb, xi, d, 6))


def test_reference_against_mpmath(small):
    """change_ref per tet (barrier orders 2 and 4, AMIPS) against the naive differences E_t(x + alpha d) - E_t(x) at 50
    digits on the same fp32 inputs, and the smoothness change of one sphere against 1/2 U(alpha)^T M U(alpha) - 1/2 U^T
    M U at 50 digits, at alpha down to 2^-23 on near-converged and inverted inputs."""
    mpmath = pytest.importorskip("mpmath")
    mp = mpmath.mp
    mp.dps = 50
    g = small.g
    rng = np.random.default_rng(11)
    for name in ("near-converged -g", "inverted", "benign shift10"):
        x32, d32 = small.inputs[name]
        p = Prep(g, x32, d32)
        tets = rng.choice(g.nt, 100, replace=False)
        x, d = x32.astype(f64), d32.astype(f64)
        for a in (1.0, 2.0 ** -8, 2.0 ** -23):
            a = float(f32(a))
            t2, t4 = tet_terms(p, a, 2), tet_terms(p, a, 4)
            for t in tets:
                idet = mp.mpf(float(g.idet[t]))
                Bm = mp.matrix(g.B[t].tolist())

                def at(al):
                    P = [[mp.mpf(float(x[v, r])) + al * mp.mpf(float(d[v, r])) for r in range(3)] for v in g.T[t]]
                    Ds = mp.matrix([[P[k + 1][r] - P[0][r] for k in range(3)] for r in range(3)])
                    J = mp.det(Ds) * idet
                    F = Ds * Bm
                    tr = sum(F[i, j] ** 2 for i in range(3) for j in range(3))
                    psi = tr / (3 * mp.cbrt(J) ** 2) - 1 if J > 0 else mp.mpf(0)
                    m = -J if J < 0 else mp.mpf(0)
                    return m, psi

                m0, p0 = at(mp.mpf(0))
                m1, p1 = at(mp.mpf(a))
                # the fp64 forms are exact to 1e-12 of the change, or to 1e-6 of the bound's unit u A (the AMIPS form's
                # two terms cancel near a similarity)
                for val, A, ref in ((t2.db[t], t2.Ab[t], m1 ** 2 - m0 ** 2), (t4.db[t], t4.Ab[t], m1 ** 4 - m0 ** 4),
                                    (t2.da[t], t2.Aa[t], p1 - p0)):
                    ref = float(ref)
                    assert abs(val - ref) <= 1e-12 * abs(ref) + 1e-6 * U * A, (name, a, t, val, ref, A)
        # smoothness of sphere 0: naive difference of energies at 50 digits
        c = 0
        vm = np.flatnonzero(g.vlab == c)
        Wc = g.W[vm][:, vm].tocoo()
        U0 = [[mp.mpf(float(p.uc[v, r])) for r in range(3)] for v in vm]
        Dd = [[mp.mpf(float(p.dr[v, r])) for r in range(3)] for v in vm]

        def half_uMu(al):
            Ua = [[U0[i][r] + al * Dd[i][r] for r in range(3)] for i in range(len(vm))]
            s = mp.mpf(0)
            for i, j, wv in zip(Wc.row, Wc.col, Wc.data):      # 1/2 u^T M u = -1/4 sum_ij w_ij |u_j - u_i|^2
                s -= mp.mpf(float(wv)) * sum((Ua[j][r] - Ua[i][r]) ** 2 for r in range(3)) / 4
            return s

        e0 = half_uMu(mp.mpf(0))
        for a in (1.0, 2.0 ** -23):
            ref = float(half_uMu(mp.mpf(a)) - e0)
            got = a * p.row1[vm].sum() + a * a * p.row2[vm].sum()
            assert abs(got - ref) <= 1e-10 * abs(ref), (name, a, got, ref)


def test_reference_taylor_limits(small):
    """With the oracle's fp64 operators: Delta E / alpha -> g^T d and (Delta E - alpha g^T d) / alpha^2 -> 1/2 d^T H d per
    term, with the oracle gradient and Hessian-vector product (test_hvp, test_hvp_amips)."""
    from test_hvp import _inverted, hvp_terms
    from test_hvp_amips import amips_hvp_terms
    pk = small.pk
    ge = Geo(pk.verts, pk.tets, exact=True)
    orc = ge.orc
    rng = np.random.default_rng(12)
    d = rng.normal(scale=0.1 * ge.h, size=pk.verts.shape).astype(f32)
    xb = perturb(pk, sigma_rel=0.02, seed=1)
    xi = _inverted(pk, seed=2)
    X = ge.X
    for x32, order in ((xb, 2), (xi, 2), (xi, 4)):
        x = x32.astype(f64)
        dd = d.astype(f64).reshape(-1)
        gs = (orc.M @ (x - X).reshape(-1))
        gb = orc.backward(1.0, x, 0.0, 1.0, order).reshape(-1)
        ga = orc.amips_backward(1.0, x, 1.0).reshape(-1)
        Mv, _, vMv, qb = hvp_terms(orc, x, dd, order)
        _, qa = amips_hvp_terms(orc, x, dd)
        lin = {"smooth": gs @ dd, "barrier": gb @ dd, "amips": ga @ dd}
        mag = {"smooth": np.abs(gs) @ np.abs(dd), "barrier": np.abs(gb) @ np.abs(dd), "amips": np.abs(ga) @ np.abs(dd)}
        quad = {"smooth": 0.5 * vMv, "barrier": 0.5 * qb.sum(), "amips": 0.5 * qa.sum()}
        for a in (2.0 ** -12, 2.0 ** -16):
            r = Ref(ge, x32, d, [a])
            val = {"smooth": r.ds[0].sum(), "barrier": r.db[order][0].sum(), "amips": r.da[0].sum()}
            for t in TERMS:
                if t == "barrier" and x32 is xb:
                    assert val[t] == 0.0            # no tet inverted at either end
                    continue
                # remainders a |quad| and a^2 |cubic|; fp64 rounding of g^T d relative to sum |g||d|
                assert abs(val[t] / a - lin[t]) <= 2 * a * abs(quad[t]) + 1e-12 * mag[t], (t, a, val[t] / a, lin[t])
                second = (val[t] - a * lin[t]) / a ** 2
                assert abs(second - quad[t]) <= 0.02 * abs(quad[t]) + 1e-12 * mag[t] / a, (t, a, second, quad[t])


def _calibration_cases(small):
    sc = single_tet_case()
    gs = Geo(sc["V"], sc["T"])
    cases = [(small.g, name, x, d) for name, (x, d) in small.inputs.items()]
    cases += [(gs, f"single tet {k}", sc["x"], v) for k, v in sc["dirs"].items()]
    return cases


def test_kappa_calibration(small):
    """The fp32 restatement against change_ref, per row and per tet, at every alpha of the GPU tests: within KAPPA / 4
    on the random inputs (benign, inverted) and on every edge family."""
    al = LADDER + POINT3
    worst = {}
    for g, name, x, d in _calibration_cases(small):
        for order in (2, 4):
            r = per_tet_ratios(g, x, d, al, order)
            for t, v in r.items():
                worst[(name, t)] = max(worst.get((name, t), 0.0), v)
    print("fp32 restatement: worst |change - change64| / (u A) per input and term (KAPPA %d):" % KAPPA)
    for (name, t), v in sorted(worst.items()):
        print(f"  {name:28s} {t:8s} {v:.3g}")
    bad = {k: v for k, v in worst.items() if not v <= KAPPA / 4}
    assert not bad, bad


def _old_bound_ok(lt, k, term, got, ref):
    """test_line_search._check's bound for one term's total at alpha_k: REL (E(x) + E(x + alpha d))."""
    if term == "smooth":
        return abs(got - ref) <= REL * (lt.s0.sum() + lt.s1[k].sum()) + 1e-12
    if term == "barrier":
        return abs(got - ref) <= REL * (lt.b0.sum() + lt.b1[k].sum()) + lt.berr[k].sum() + 1e-12
    return abs(got - ref) <= REL * (lt.a0.sum() + lt.a1[k].sum()) + 1e-12


MUTATIONS = {   # regression: (mutation, input of x, input of d, term, alphas)
    "plain_tet barrier": ("plain_tet", "inverted", "inverted", "barrier", LADDER[8:]),
    "plain_tet amips": ("plain_tet", "benign", "benign", "amips", LADDER[8:]),
    "plain_smooth": ("plain_smooth", "benign", "benign", "smooth", LADDER[8:]),
    "no_shift": ("no_shift", "near-converged shift10", "near-converged shift10", "smooth", LADDER[16:]),
    "corner_dF": ("corner_dF", "inverted", "benign d+1e+04h", "barrier", LADDER[12:]),
}


@pytest.mark.parametrize("case", list(MUTATIONS))
def test_regressions_fail_the_new_bound(small, case):
    """Each regression passes test_line_search's energy-relative bound on the total at every alpha used and fails this
    file's bound by more than 100x at its finest level: per tet for the tet terms (as the single-tet handle enforces
    it), per sphere for the smoothness (its per-row split is the kernel's own).  The margin is the largest |change_mut -
    change64| / (KAPPA u A + u |change64| + allowance); the unmutated restatement stays within the bound."""
    mut, xname, dname, term, al = MUTATIONS[case]
    g = small.g
    x32, d32 = small.inputs[xname][0], small.inputs[dname][1]
    order = 2
    ref = Ref(g, x32, d32, al)
    lt = line_terms(g.orc, x32.astype(f64), d32.astype(f64), np.asarray(np.asarray(al, f32), f64), order, 1.0)
    j = TERMS.index(term) + 1
    val, A, allow = ref.term(j, order, 1.0)
    p = Prep(g, x32, d32)

    def over(err, bound):
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(err == 0, 0.0, np.abs(err) / bound)

    def margins(m):
        """(finest-level margin, total margin, totals [K])"""
        ds, db, da = reenact_fp32(g, x32, d32, al, order, m)
        if term == "smooth":
            per = np.array([_sphere_sum(g.vlab, g.S, ds[k]) for k in range(len(al))])
            fine = over(per - val, KAPPA * U * A + U * np.abs(val) + allow).max()
            tot = per.sum(1)
        else:
            fine = 0.0
            for k, a in enumerate(ref.alphas):
                t = tet_terms(p, a, order)
                got, v, sc, alw = (db[k], t.db, t.Ab, t.allow_b) if term == "barrier" else (da[k], t.da, t.Aa, 0.0)
                ok = ~t.amb_a if term == "amips" else np.ones(g.nt, bool)
                fine = max(fine, over(got - v, KAPPA * U * sc + U * np.abs(v) + alw)[ok].max())
            tot = (db if term == "barrier" else da).sum(1)
        r64 = val.sum(1)
        return fine, over(tot - r64, KAPPA * U * A.sum(1) + U * np.abs(r64) + allow.sum(1)).max(), tot

    fine, total, got = margins(mut)
    fine0, total0, _ = margins(None)
    for k in range(len(al)):
        assert _old_bound_ok(lt, k, term, got[k], val[k].sum()), (case, al[k], got[k], val[k].sum())
    print(f"{case} on x {xname}, d {dname}, alpha 2^-{-np.log2(al[0]):.0f}..2^-23: margin {fine:.3g}x "
          f"({'sphere' if term == 'smooth' else 'tet'}), {total:.3g}x (total); unmutated {fine0:.3g}, {total0:.3g}")
    assert fine0 <= 1.0 and total0 <= 1.0
    assert fine >= 100.0, (case, fine)


def test_unshifted_d_edges_are_exact(small):
    """Staging d without - d_ref changes nothing the tets see: the edge differences of two fp32 components are exact
    (Sterbenz) or correctly rounded either way, so on a direction with a large per-sphere translation the fp32 edges
    are bitwise those of the staged d - d_r.  (corner_dF above is the form in which a translation does enter a rounded
    sum.)"""
    g = small.g
    _, d32 = small.inputs["benign d+1e+04h"]
    w = d32 - d32[g.rv]
    for k in (1, 2, 3):
        assert np.array_equal(d32[g.T[:, k]] - d32[g.T[:, 0]], w[g.T[:, k]] - w[g.T[:, 0]])


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
    return ext.TetSpheres(np.ascontiguousarray(V, f32).reshape(-1), np.ascontiguousarray(T, np.int32).reshape(-1), **kw)


_GPU = {}


def gpu_mesh(name):
    """(Geo, {input: (x32, d32)}) of a GPU mesh, built once."""
    if name not in _GPU:
        if name == "single":
            sc = single_tet_case()
            g = Geo(sc["V"], sc["T"])
            ins = {f"single {k}": (sc["x"], v) for k, v in sc["dirs"].items()}
            _GPU[name] = (g, ins, sc)
        else:
            from test_line_search import _mesh
            V, T, _, xs, d = _mesh(name)
            g = Geo(V, T)
            ins = inputs(g, xs["benign"], xs["inverted"], d, 40)
            if "stretched" in xs:
                ins["stretched"] = (np.ascontiguousarray(xs["stretched"], f32), d)
            _GPU[name] = (g, ins, None)
    return _GPU[name]


_PREPS, _REFS = {}, {}


def gpu_ref(name, inp, alphas):
    key = (name, inp, tuple(alphas))
    if key not in _REFS:
        g, ins, _ = gpu_mesh(name)
        x, d = ins[inp]
        if (name, inp) not in _PREPS:
            _PREPS[(name, inp)] = Prep(g, x, d)
        _REFS[key] = Ref(g, x, d, alphas, _PREPS[(name, inp)])
    return _REFS[key]


def _launch(sp, x, d, alphas, order, c3):
    torch = _torch()
    r = sp.line_search(torch.from_numpy(x).cuda(), torch.from_numpy(d).cuda(), alphas, C1, C2, order, c3=c3, per_sphere=True)
    torch.cuda.synchronize()
    return (r.delta.cpu().numpy().astype(f64), float(r.max_step), r.sphere_delta.cpu().numpy().astype(f64),
            r.sphere_max_step.cpu().numpy())


WORST = {}


def check_launch(name, inp, alphas, order, c3, out):
    """Every term per sphere and in total, and the total column, against change_ref within the bound; records the worst
    ratio per input family and term."""
    delta, _, sd, _ = out
    ref = gpu_ref(name, inp, alphas)
    g = gpu_mesh(name)[0]
    fam = inp
    amb = ref.amb_a if c3 else np.zeros_like(ref.amb_a)
    tot_v, tot_A, tot_allow = 0.0, 0.0, 0.0
    for j, term, c in ((1, "smooth", C1), (2, "barrier", C2), (3, "amips", c3)):
        val, A, allow = ref.term(j, order, c3)
        ok = ~amb if j == 3 else np.ones_like(amb)
        rs = ratio(sd[:, :, j].T - val, val, A, allow)                     # [K, S]
        bad = np.argwhere(ok & (rs > KAPPA))
        assert not len(bad), (name, inp, order, c3, term, [(alphas[k], s, rs[k, s], sd[s, k, j], val[k, s]) for k, s in bad[:6]])
        if c3 == 0 and j == 3:
            assert not sd[:, :, 3].any() and not delta[:, 3].any()
        allk = ~amb.any(axis=1) if j == 3 else np.ones(len(alphas), bool)
        rt = ratio(delta[:, j] - val.sum(1), val.sum(1), A.sum(1), allow.sum(1))
        assert np.all(rt[allk] <= KAPPA), (name, inp, order, c3, term, rt)
        key = (name, fam, term)
        cur = [rs[ok].max() if ok.any() else 0.0, rt[allk].max() if allk.any() else 0.0]
        WORST[key] = max(WORST.get(key, 0.0), *cur)
        tot_v = tot_v + c * val
        tot_A = tot_A + c * A
        tot_allow = tot_allow + c * allow
    # the total column: c1 ds + c2 db + c3 da against fp64, per sphere and in total
    allk = ~amb.any(axis=1)
    rs = ratio(sd[:, :, 0].T - tot_v, tot_v, tot_A, tot_allow)
    assert not np.any((rs > KAPPA) & ~amb), (name, inp, order, c3, "total")
    rt = ratio(delta[:, 0] - tot_v.sum(1), tot_v.sum(1), tot_A.sum(1), tot_allow.sum(1))
    assert np.all(rt[allk] <= KAPPA), (name, inp, order, c3, "total", rt)
    WORST[(name, fam, "total")] = max(WORST.get((name, fam, "total"), 0.0), rs[~amb].max() if (~amb).any() else 0.0)
    return ref, tot_v, tot_A, tot_allow


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nline search change: worst |change_gpu - change64| / (u A) per mesh, input family and term (KAPPA %d):" % KAPPA)
        for (m, fam, t), v in sorted(WORST.items()):
            print(f"  {m:12s} {fam:22s} {t:8s} {v:.3g}")


def run_mesh(ext, name, kw, orders_c3=((2, 0.0), (2, C3), (4, 0.0), (4, C3))):
    g, ins, _ = gpu_mesh(name)
    sp = _handle(ext, g.V32, g.T, enable_amips=True, **kw)
    assert sp.info["n_components"] == g.S
    for inp, (x, d) in ins.items():
        for alphas in LAUNCHES:
            for order, c3 in orders_c3:
                check_launch(name, inp, alphas, order, c3, _launch(sp, x, d, alphas, order, c3))
    return sp


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(warps_per_cta=8), dict(deterministic=True)], ids=["w16", "w8", "det"])
def test_staged_pack(ext, kw):
    sp = run_mesh(ext, "pack64x4096", kw)
    assert sp.info["mode_global"] == 0


@pytest.mark.gpu
def test_a_veg_global(ext):
    sp = run_mesh(ext, "a_veg", dict(force_global=True))
    assert sp.info["mode_global"] == 1


@pytest.mark.gpu
def test_shuffled_ids_with_orphans(ext):
    g = gpu_mesh("shuffled")[0]
    assert (~g.used).sum() == 500
    run_mesh(ext, "shuffled", dict())


@pytest.mark.gpu
@pytest.mark.parametrize("mesh,kw", plan_shape_cases(deterministic=False))
def test_line_search_plan_shapes(ext, mesh, kw):
    """The changes on the plans only these meshes produce (assert_plan_shape): the staged direction of whole-area
    segments, the direction prefetched past the segment table, the pole's ring-wrapping row block."""
    sp = run_mesh(ext, mesh, kw)
    check_handle_plan_shape(mesh, sp, kw, enable_amips=True)


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(deterministic=True)], ids=["default", "det"])
def test_single_tets(ext, kw):
    """Every tet its own sphere: sphere_delta is a per-tet check, at J near 0 (+-1e-2 .. +-2^-20), needles and J = 0
    exactly, along directions that push J through 0 and pull it away."""
    g, ins, sc = gpu_mesh("single")
    assert g.S == g.nt
    run_mesh(ext, "single", kw)
    # the families reach both signs and both classifications of J = 0
    p = Prep(g, sc["x"], sc["dirs"]["push"])
    assert (p.J0 == 0).sum() >= 6 and (p.J0 < 0).sum() >= 20 and (p.J0 > 0).sum() >= 20


@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", [("pack64x4096", dict()), ("pack64x4096", dict(deterministic=True)),
                                     ("a_veg", dict(force_global=True)), ("shuffled", dict())],
                         ids=["pack", "pack-det", "a_veg-global", "shuffled"])
def test_translation_gives_exact_zeros(ext, name, kw):
    """d = a per-sphere translation: the staged d - d_ref is exactly 0, so every term of every sphere is exactly 0 at
    every alpha and no tet has a root (step +inf), at 1e2 h and 1e4 h, on the benign and the shifted input."""
    g, ins, _ = gpu_mesh(name)
    sp = _handle(ext, g.V32, g.T, enable_amips=True, **kw)
    for s in (1e2, 1e4, 1.0):
        t = sphere_translations(g, s * g.h, 77).astype(f32)
        for inp in ("benign", "benign shift10"):
            x = ins[inp][0]
            for alphas in LAUNCHES:
                for order, c3 in ((2, C3), (4, 0.0)):
                    delta, step, sd, ss = _launch(sp, x, t, alphas, order, c3)
                    assert not delta.any() and not sd.any(), (name, s, inp, order)
                    assert step == np.inf and np.all(ss == np.inf)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["pack64x4096", "shuffled"])
def test_armijo_sign_agrees_with_fp64(ext, name):
    """Along -g64 on the benign and near-converged inputs: wherever the fp64 Armijo margin Delta E + sigma alpha |g|^2
    of a sphere exceeds the bound, the kernel's total column gives it the same sign.  Prints the smallest alpha at
    which every sphere still agrees."""
    g, ins, _ = gpu_mesh(name)
    sp = _handle(ext, g.V32, g.T, enable_amips=True)
    for inp in ("benign -g", "near-converged -g"):
        x, d = ins[inp]
        gd = _sphere_sum(g.vlab, g.S, _dot(oracle_gradient(g, x), d.astype(f64)))     # g^T d < 0 per sphere
        assert np.all(gd < 0)
        agree_all = []
        for alphas in LAUNCHES[:3]:
            out = _launch(sp, x, d, alphas, 2, C3)
            ref, tot_v, tot_A, tot_allow = check_launch(name, inp, alphas, 2, C3, out)
            al = ref.alphas[:, None]
            m64 = tot_v - SIGMA * al * gd[None]
            mg = out[2][:, :, 0].T - SIGMA * al * gd[None]
            bound = KAPPA * U * tot_A + U * np.abs(tot_v) + tot_allow
            sure = (np.abs(m64) > bound) & ~ref.amb_a
            assert np.all(np.sign(mg[sure]) == np.sign(m64[sure])), (name, inp)
            agree_all += list(zip(ref.alphas, np.all(np.sign(mg) == np.sign(m64), axis=1), sure.mean(axis=1)))
        agree_all.sort(key=lambda t: -t[0])
        smallest = None
        for a, ok, _ in agree_all:
            if not ok:
                break
            smallest = a
        print(f"{name} {inp}: every sphere's Armijo sign agrees with fp64 down to alpha = {smallest}; "
              f"decided (|margin| > bound) at alpha 2^-23: {agree_all[-1][2]:.0%} of the spheres")
