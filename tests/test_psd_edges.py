"""The projected tet Hessians of psd_project_kernel (tsb_psd.cu) at the edges of its signed SVD, tet by tet.

CPU: project_reenact, the kernel's projection restated in fp64 numpy operation for operation (Jacobi eigen-system of
F^T F, sort, proper V, one one-sided Jacobi sweep on the columns of F V, Gram-Schmidt, the closed forms, the clamp of A),
its 30 stored floats rounded to fp32, against numpy.linalg.eigh of the 9 x 9 F-space Hessian, on random F (calibrating
KAPPA), _newton_model's cases, needles, a collapsing plane, equal singular values with a negative s_3, a large stretch
and a uniformly tiny F, in both signs of det F and rounded to fp32; the fp64 stage alone; the algorithm without the
one-sided sweep fails the needles; apply_reenact, psd_apply_kernel's fp32 product, and its curvature.  GPU: a handle of
disjoint single-tet components (unit right tets with B = I and a generic rest tet far from the origin), so every tet's F
is chosen exactly and each tet's corners carry its product alone (c1 = 0), against the fp64 projection; the curvature
record; flat and collapsed tets; AMIPS at rotations; inverted tets with AMIPS on."""
import numpy as np
import pytest

from _newton_model import C3, COEF, _cases, _cuda, _handle, _rot, _torch, ext  # noqa: F401
from test_hess_diag import psi_hessians

U32 = 2.0 ** -24                # fp32 unit roundoff
FLT_MIN = 2.0 ** -126           # smallest normal fp32: the floor of an operator entry's absolute error
# |P - P(H)|_max <= KAPPA (u lambda_max + FLT_MIN) per tet for the stored operator, and the same with the product's
# magnitude for a corner product (test_kappa_calibration: worst ratio on random F, which must stay within KAPPA / 4)
KAPPA = 16
KAPPA_Q = 1                     # the fp32 curvature q = Dh : D' >= -KAPPA_Q u lambda_max |dF|^2 (test_curvature_floor)
FP64_STAGE = 1e-9               # the operator before fp32 rounding, relative to lambda_max


# ---------------------------------------------------------------------------------------------------------------------
# psd_project_kernel and psd_apply_kernel in numpy, vectorised over tets


def _jacobi_rot(S, V, p, q):
    """tsb_jacobi.cuh's jacobi_rot on symmetric S [T, 3, 3]: zero S_pq and rotate columns p and q of V."""
    r = 3 - p - q
    app, aqq, apq, apr, aqr = S[:, p, p].copy(), S[:, q, q].copy(), S[:, p, q].copy(), S[:, p, r].copy(), S[:, q, r].copy()
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        theta = (aqq - app) / (2.0 * apq)
        t = np.copysign(1.0, theta) / (np.abs(theta) + np.sqrt(theta * theta + 1.0))
    t = np.where(apq != 0.0, t, 0.0)            # apq == 0: no rotation
    c = 1.0 / np.sqrt(t * t + 1.0)
    s = t * c
    S[:, p, p] = app - t * apq
    S[:, q, q] = aqq + t * apq
    S[:, p, q] = S[:, q, p] = 0.0
    S[:, p, r] = S[:, r, p] = c * apr - s * aqr
    S[:, q, r] = S[:, r, q] = s * apr + c * aqr
    vp, vq = V[:, :, p].copy(), V[:, :, q].copy()
    c, s = c[:, None], s[:, None]
    V[:, :, p] = c * vp - s * vq
    V[:, :, q] = s * vp + c * vq


def sym_eig(S):
    """sym_eig: 8 cyclic sweeps in the kernel's rotation order (its early exit when S is diagonal changes nothing)."""
    S = S.copy()
    V = np.broadcast_to(np.eye(3), S.shape).copy()
    for _ in range(8):
        for p, q in ((0, 1), (0, 2), (1, 2)):
            _jacobi_rot(S, V, p, q)
    return S[:, [0, 1, 2], [0, 1, 2]].copy(), V


def _swap(mask, ev, cols, a, b):
    """Swap entries a and b of ev and columns a and b of every matrix in cols where mask."""
    ev[mask, a], ev[mask, b] = ev[mask, b], ev[mask, a].copy()
    for M in cols:
        M[mask, :, a], M[mask, :, b] = M[mask][:, :, b], M[mask][:, :, a].copy()


def _sort_desc(ev, cols):
    for a, b in ((0, 1), (1, 2), (0, 1)):
        _swap(ev[:, a] < ev[:, b], ev, cols, a, b)


def _det3(F):
    return (F[:, 0, 0] * (F[:, 1, 1] * F[:, 2, 2] - F[:, 1, 2] * F[:, 2, 1]) - F[:, 0, 1] * (F[:, 1, 0] * F[:, 2, 2] - F[:, 1, 2] * F[:, 2, 0])
            + F[:, 0, 2] * (F[:, 1, 0] * F[:, 2, 1] - F[:, 1, 1] * F[:, 2, 0]))


def _dot(a, b):
    return a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1] + a[:, 2] * b[:, 2]


def _cross(a, b):
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)


def _one_sided_sweep(W, V):
    """One one-sided (Hestenes) Jacobi sweep: per column pair of W = F V, the rotation that makes w_p and w_q
    orthogonal, from their own dot products, applied to W and V."""
    for p, q in ((0, 1), (0, 2), (1, 2)):
        wp, wq = W[:, :, p].copy(), W[:, :, q].copy()
        al, be, ga = _dot(wp, wp), _dot(wq, wq), _dot(wp, wq)
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            theta = (be - al) / (2.0 * ga)
            t = np.copysign(1.0, theta) / (np.abs(theta) + np.sqrt(theta * theta + 1.0))
        t = np.where(ga != 0.0, t, 0.0)
        c = (1.0 / np.sqrt(t * t + 1.0))[:, None]
        s = t[:, None] * c
        W[:, :, p], W[:, :, q] = c * wp - s * wq, s * wp + c * wq
        vp, vq = V[:, :, p].copy(), V[:, :, q].copy()
        V[:, :, p], V[:, :, q] = c * vp - s * vq, s * vp + c * vq


PK = (2, 1, 0)                  # the third index of the pairs (0, 1), (0, 2), (1, 2)
PAIRS = ((0, 1), (0, 2), (1, 2))


def project_reenact(F, order, amips, refine=True):
    """psd_project_kernel on F [T, 3, 3] (fp64): (kind, fp64 operator, the same rounded to fp32).  kind 0 inactive, 1
    barrier (J < 0), 2 AMIPS (J > 0 and amips); an operator is a dict U, V [T, 3, 3] (columns u_i, v_i), Ap (A+,
    [T, 3, 3]), ls, la ([T, 3], clamped), meaningful on active tets.  refine=False: the algorithm before the one-sided
    sweep."""
    F = np.asarray(F, np.float64)
    T = len(F)
    J = _det3(F)
    kind = np.where(J < 0.0, 1, np.where((J > 0.0) & bool(amips), 2, 0))
    ok = kind != 0
    Fa = np.where(ok[:, None, None], F, np.eye(3))              # inactive tets: any finite input, result unused
    Ja = np.where(ok, J, 1.0)
    S = sum(Fa[:, r, :, None] * Fa[:, r, None, :] for r in range(3))
    ev, V = sym_eig(S)
    _sort_desc(ev, [V])
    neg = _det3(V) < 0.0
    V[neg, :, 2] *= -1.0
    W = sum(Fa[:, :, c, None] * V[:, None, c, :] for c in range(3))       # W[:, r, i] = (F v_i)_r
    if refine:
        _one_sided_sweep(W, V)
        n2 = np.stack([_dot(W[:, :, i], W[:, :, i]) for i in range(3)], axis=1)
        _sort_desc(n2, [V, W])
        neg = _det3(V) < 0.0
        V[neg, :, 2] *= -1.0
        W[neg, :, 2] *= -1.0
    w = [W[:, :, i] for i in range(3)]
    sg0 = np.sqrt(_dot(w[0], w[0]))
    u0 = w[0] / sg0[:, None]
    pr = _dot(u0, w[1])
    u1 = w[1] - pr[:, None] * u0
    sg1 = np.sqrt(_dot(u1, u1))
    fb = ~(sg1 > 1e-150 * sg0)
    if fb.any():                                # any unit vector orthogonal to u_1, from the axis it is least along
        a0, a1, a2 = np.abs(u0[:, 0]), np.abs(u0[:, 1]), np.abs(u0[:, 2])
        ax = np.where(a0 < a1, np.where(a0 < a2, 0, 2), np.where(a1 < a2, 1, 2))
        u1 = np.where(fb[:, None], _cross(u0, np.eye(3)[ax]), u1)
    u1 = u1 * (1.0 / np.sqrt(_dot(u1, u1)))[:, None]
    u2 = _cross(u0, u1)
    sg = np.stack([sg0, sg1, Ja / (sg0 * sg1)], axis=1)

    A = np.zeros((T, 3, 3))
    ls, la = np.zeros((T, 3)), np.zeros((T, 3))
    with np.errstate(all="ignore"):
        # barrier
        m = -Ja
        d1 = -2.0 * m if order == 2 else -4.0 * m * m * m
        d2 = np.full(T, 2.0) if order == 2 else 12.0 * m * m
        g = np.stack([sg[:, 1] * sg[:, 2], sg[:, 0] * sg[:, 2], sg[:, 0] * sg[:, 1]], axis=1)
        Ab = np.stack([np.stack([d2 * g[:, i] * g[:, j] + (0.0 if i == j else d1 * sg[:, 3 - i - j]) for j in range(3)], 1)
                       for i in range(3)], 1)
        lsb = np.stack([-d1 * sg[:, k] for k in PK], 1)
        lab = np.stack([d1 * sg[:, k] for k in PK], 1)
        # AMIPS
        cb = np.cbrt(Ja)
        j23 = cb * cb
        al = 2.0 / (3.0 * j23)
        ga = 2.0 * (sg[:, 0] * sg[:, 0] + sg[:, 1] * sg[:, 1] + sg[:, 2] * sg[:, 2]) / (9.0 * j23)
        Aa = np.stack([np.stack([-al / 3.0 + (5.0 / 3.0) * ga / (sg[:, i] * sg[:, i]) if i == j else
                                 -(2.0 / 3.0) * al * (sg[:, i] / sg[:, j] + sg[:, j] / sg[:, i]) + (2.0 / 3.0) * ga / (sg[:, i] * sg[:, j])
                                 for j in range(3)], 1) for i in range(3)], 1)
        r = np.stack([ga / (sg[:, i] * sg[:, j]) for i, j in PAIRS], 1)
    bar = (kind == 1)[:, None]
    A = np.where(bar[:, :, None], Ab, Aa)
    ls, la = np.where(bar, lsb, al[:, None] + r), np.where(bar, lab, al[:, None] - r)
    A = np.where(ok[:, None, None], A, 0.0)
    lam, Q = sym_eig(A)
    lam = np.maximum(lam, 0.0)
    Ap = np.stack([np.stack([lam[:, 0] * Q[:, a, 0] * Q[:, b, 0] + lam[:, 1] * Q[:, a, 1] * Q[:, b, 1] + lam[:, 2] * Q[:, a, 2] * Q[:, b, 2]
                             for b in range(3)], 1) for a in range(3)], 1)
    op = dict(U=np.stack([u0, u1, u2], axis=2), V=V, Ap=Ap, ls=np.maximum(ls, 0.0), la=np.maximum(la, 0.0))
    op32 = {k: v.astype(np.float32) for k, v in op.items()}
    return kind, op, op32


def _pair_rule(Dh, Ap, ls, la):
    """D' from Dh (any float type, [..., 3, 3]): diag D' = A+ diag Dh, and per pair s, a = (Dh_ij +- Dh_ji) / 2, D'_ij =
    ls s + la a, D'_ji = ls s - la a (psd_apply_kernel's order)."""
    Dp = np.zeros_like(Dh)
    for i in range(3):
        Dp[..., i, i] = Ap[..., i, 0] * Dh[..., 0, 0] + Ap[..., i, 1] * Dh[..., 1, 1] + Ap[..., i, 2] * Dh[..., 2, 2]
    half = Dh.dtype.type(0.5)
    for P, (i, j) in enumerate(PAIRS):
        s, a = half * (Dh[..., i, j] + Dh[..., j, i]), half * (Dh[..., i, j] - Dh[..., j, i])
        Dp[..., i, j] = ls[..., P] * s + la[..., P] * a
        Dp[..., j, i] = ls[..., P] * s - la[..., P] * a
    return Dp


def op_matrix(op):
    """[T, 9, 9] fp64 matrix (row-major vec F) of dF -> U D'(U^T dF V) V^T for an operator (fp64 or fp32 entries)."""
    o = {k: np.asarray(v, np.float64) for k, v in op.items()}
    E = np.eye(9).reshape(9, 3, 3)
    Dh = np.einsum("tri,qrc,tcj->tqij", o["U"], E, o["V"])
    Dp = _pair_rule(Dh, o["Ap"][:, None], o["ls"][:, None], o["la"][:, None])
    P = np.einsum("tri,tqij,tcj->tqrc", o["U"], Dp, o["V"]).reshape(-1, 9, 9)
    return P.transpose(0, 2, 1)


def apply_reenact(op32, B, vs, wt):
    """psd_apply_kernel in fp32 on active tets: corners [T, 4, 3] of wt P[dF], dF = dDs B, and q = Dh : D' [T].
    B [T, 3, 3] and vs [T, 4, 3] (the corner values of v) as fp32."""
    f = np.float32
    B, vs, wt = np.asarray(B, f), np.asarray(vs, f), f(wt)
    U, V = op32["U"], op32["V"]
    e = [vs[:, k + 1] - vs[:, 0] for k in range(3)]                        # [T, 3] each
    dF = e[0][:, :, None] * B[:, 0, None, :] + e[1][:, :, None] * B[:, 1, None, :] + e[2][:, :, None] * B[:, 2, None, :]
    Tm = U[:, 0, :, None] * dF[:, 0, None, :] + U[:, 1, :, None] * dF[:, 1, None, :] + U[:, 2, :, None] * dF[:, 2, None, :]
    Dh = Tm[:, :, 0, None] * V[:, None, 0, :] + Tm[:, :, 1, None] * V[:, None, 1, :] + Tm[:, :, 2, None] * V[:, None, 2, :]
    Dp = _pair_rule(Dh, op32["Ap"], op32["ls"], op32["la"])
    q = np.zeros(len(B), f)
    for i in range(3):
        for j in range(3):
            q = q + Dh[:, i, j] * Dp[:, i, j]
    W = U[:, :, 0, None] * Dp[:, None, 0, :] + U[:, :, 1, None] * Dp[:, None, 1, :] + U[:, :, 2, None] * Dp[:, None, 2, :]
    Pm = W[:, :, 0, None] * V[:, None, :, 0] + W[:, :, 1, None] * V[:, None, :, 1] + W[:, :, 2, None] * V[:, None, :, 2]
    g = np.zeros((len(B), 4, 3), f)
    for k in range(3):
        c = wt * (Pm[:, :, 0] * B[:, k, None, 0] + Pm[:, :, 1] * B[:, k, None, 1] + Pm[:, :, 2] * B[:, k, None, 2])
        g[:, k + 1] = c
        g[:, 0] = g[:, 0] - c
    return g, q


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference


def eigh_reference(F, kind, order):
    """[T, 9, 9] fp64 projections P(H) of each tet's active term (zero on inactive tets) and lambda_max of H."""
    Hb = psi_hessians(F, order=order)
    Ha = psi_hessians(F, amips=True)
    H = np.where((kind == 1)[:, None, None], Hb, np.where((kind == 2)[:, None, None], Ha, 0.0))
    w, Q = np.linalg.eigh(0.5 * (H + H.transpose(0, 2, 1)))
    return np.einsum("tij,tj,tkj->tik", Q, np.maximum(w, 0.0), Q), np.maximum(w.max(axis=1), 0.0)


def reference_corners(P, B, vs, wt):
    """fp64 corners [T, 4, 3] of wt P[dF] with dF = dDs B, and the magnitude wt |B|_F |dF|abs|_F of each product."""
    B, vs = np.asarray(B, np.float64), np.asarray(vs, np.float64)
    e = vs[:, 1:] - vs[:, :1]                                               # [T, 3 (k), 3 (r)]
    dF = np.einsum("tkr,tkc->trc", e, B)
    Y = np.einsum("tij,tj->ti", P, dF.reshape(-1, 9)).reshape(-1, 3, 3)
    c = wt * np.einsum("trc,tkc->tkr", Y, B)
    g = np.concatenate([-c.sum(axis=1, keepdims=True), c], axis=1)
    mag = wt * np.linalg.norm(B, axis=(1, 2)) * np.linalg.norm(np.einsum("tkr,tkc->trc", np.abs(e), np.abs(B)), axis=(1, 2))
    return g, mag, dF


def f32(F):
    return np.asarray(F, np.float32).astype(np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# cases


def _diag_rot(rng, s):
    return _rot(rng) @ np.diag(s) @ _rot(rng).T


NEEDLES = (1e-4, 1e-5, 1e-6, 1e-7)


def exact_needle(a, b):
    """F with exact fp32 entries, singular values ~ (sqrt 3, a sqrt(2/3), b / sqrt 2): unit right tet edges (1, 0, 0),
    (1, a, 0) and (1, 0, b)."""
    return np.array([[1.0, 1.0, 1.0], [0.0, a, 0.0], [0.0, 0.0, b]])


def edge_cases(rng, gpu=False):
    """{family: [F, ...]} in fp64, both signs of det F (the sign of s_3 flipped), rounded to fp32.  gpu=False adds the
    cases whose AMIPS operator leaves the fp32 range (s_2 / s_1 ~ 1e-8 and below)."""
    fam = {"newton_psd": [F for _, F in _cases(rng)]}
    fam["needle"] = [_diag_rot(rng, [1.0, s, s / 100]) for s in NEEDLES for _ in range(3)]
    fam["needle"] += [exact_needle(2.0 ** -k, 2.0 ** -(k + 7)) for k in (13, 17, 20, 23)]
    if not gpu:
        fam["needle"] += [_diag_rot(rng, [1.0, 1e-8, 1e-10]) for _ in range(3)] + [exact_needle(2.0 ** -30, 2.0 ** -40)]
    fam["plane"] = [_diag_rot(rng, [1.0, 0.999, 1e-7]) for _ in range(3)]
    fam["equal"] = [_diag_rot(rng, s) for s in ([1.3, 0.8, -0.8], [0.9, 0.9, -0.9]) for _ in range(2)]
    fam["stretch"] = [_diag_rot(rng, [1e3, 1.0, 1e-3]) for _ in range(3)]
    fam["tiny"] = [1e-6 * _diag_rot(rng, [1.2, 0.9, 0.7]) for _ in range(3)]
    flip = np.diag([1.0, 1.0, -1.0])
    return {k: f32(np.stack([G for F in v for G in (F, F @ flip)])) for k, v in fam.items()}


def random_F(rng, n):
    """Random F for the calibration: Gaussian, and rotations times log-uniform singular values in [1e-3, 1e3] with a
    random sign of s_3, rounded to fp32."""
    G = rng.standard_normal((n // 2, 3, 3))
    s = 10.0 ** rng.uniform(-3, 3, (n - n // 2, 3)) * np.stack([np.ones(n - n // 2)] * 2 + [rng.choice([-1.0, 1.0], n - n // 2)], 1)
    R = np.stack([_diag_rot(rng, si) for si in s])
    return f32(np.concatenate([G, R]))


TERMS = {"barrier2": (2, False), "barrier4": (4, False), "amips": (2, True)}


def _term_cases(F, term):
    """The tets of F where the term is the active one: J < 0 for the barrier, J > 0 for AMIPS."""
    J = _det3(F)
    return F[J > 0] if TERMS[term][1] else F[J < 0]


def op_ratio(F, term, refine=True):
    """Per tet: (|P64 - P(H)|_max / lambda_max, |P32 - P(H)|_max / (u lambda_max + FLT_MIN)) of the re-enactment."""
    order, amips = TERMS[term]
    kind, op, op32 = project_reenact(F, order, amips, refine)
    assert (kind == (2 if amips else 1)).all()
    P, lmax = eigh_reference(F, kind, order)
    e64 = np.abs(op_matrix(op) - P).max(axis=(1, 2)) / lmax
    e32 = np.abs(op_matrix(op32) - P).max(axis=(1, 2)) / (U32 * lmax + FLT_MIN)
    return e64, e32


# ---------------------------------------------------------------------------------------------------------------------
# CPU


@pytest.mark.parametrize("term", list(TERMS))
def test_kappa_calibration(term):
    """Random F: the fp32 operator within KAPPA / 4, the fp64 stage within FP64_STAGE."""
    F = _term_cases(random_F(np.random.default_rng(11), 4000), term)
    e64, e32 = op_ratio(F, term)
    print(f"{term}: {len(F)} random F, worst |P32 - P(H)| / (u lambda_max) = {e32.max():.3g} (KAPPA {KAPPA}), "
          f"fp64 stage {e64.max():.2e}")
    assert e64.max() <= FP64_STAGE
    assert e32.max() <= KAPPA / 4


@pytest.mark.parametrize("term", list(TERMS))
def test_edge_cases_against_eigh(term):
    """Every case family: the fp64 stage within FP64_STAGE of P(H), the stored fp32 operator within KAPPA."""
    fam = edge_cases(np.random.default_rng(5))
    for name, F in fam.items():
        F = _term_cases(F, term)
        if not len(F):
            continue
        e64, e32 = op_ratio(F, term)
        print(f"{term} {name}: {len(F)} tets, worst |P32 - P(H)| / (u lambda_max) {e32.max():.3g}, fp64 stage {e64.max():.2e}")
        assert e64.max() <= FP64_STAGE, (name, e64)
        assert e32.max() <= KAPPA, (name, e32)


def test_old_algorithm_misses_needles():
    """Without the one-sided sweep (V from F^T F alone) the needles with s_2 / s_1 <= 1e-6 fail the bound: eigenvalues of
    F^T F below ~ eps s_1^2 are lost, v_2 and v_3 mix and the clamped eigenvalues land in the wrong frame.  With it they
    pass."""
    rng = np.random.default_rng(5)
    groups = {f"s2/s1={s:g}": f32(np.stack([_diag_rot(rng, [1.0, s, s / 100]) for _ in range(3)])) for s in (1e-6, 1e-7)}
    groups["exact 2^-20, 2^-27"] = f32(exact_needle(2.0 ** -20, 2.0 ** -27)[None])
    groups["exact 2^-23, 2^-30"] = f32(exact_needle(2.0 ** -23, 2.0 ** -30)[None])
    flip = np.diag([1.0, 1.0, -1.0])
    for name, F in groups.items():
        F = np.concatenate([F, F @ flip])
        for term in ("barrier2", "amips"):
            Ft = _term_cases(F, term)
            old64, old = op_ratio(Ft, term, refine=False)
            _, new = op_ratio(Ft, term)
            print(f"{term} {name}: worst ratio without the sweep {old.max():.3g}, with it {new.max():.3g}")
            assert old.max() > KAPPA and old64.max() > FP64_STAGE, (term, name, old)
            assert new.max() <= KAPPA, (term, name, new)


def _host_B(X, tets):
    """tsb_pcg_enable_psd's B = Dm^-1 (fp64 cofactors of the fp32 rest edges, stored as fp32), [T, 3, 3]."""
    X = np.asarray(X, np.float32).astype(np.float64)
    P = X[np.asarray(tets)]
    D = (P[:, 1:] - P[:, :1]).transpose(0, 2, 1)                            # D[r][k]
    c00 = D[:, 1, 1] * D[:, 2, 2] - D[:, 1, 2] * D[:, 2, 1]
    c01 = D[:, 1, 2] * D[:, 2, 0] - D[:, 1, 0] * D[:, 2, 2]
    c02 = D[:, 1, 0] * D[:, 2, 1] - D[:, 1, 1] * D[:, 2, 0]
    det = D[:, 0, 0] * c00 + D[:, 0, 1] * c01 + D[:, 0, 2] * c02
    inv = np.stack([
        np.stack([c00, D[:, 0, 2] * D[:, 2, 1] - D[:, 0, 1] * D[:, 2, 2], D[:, 0, 1] * D[:, 1, 2] - D[:, 0, 2] * D[:, 1, 1]], 1),
        np.stack([c01, D[:, 0, 0] * D[:, 2, 2] - D[:, 0, 2] * D[:, 2, 0], D[:, 0, 2] * D[:, 1, 0] - D[:, 0, 0] * D[:, 1, 2]], 1),
        np.stack([c02, D[:, 0, 1] * D[:, 2, 0] - D[:, 0, 0] * D[:, 2, 1], D[:, 0, 0] * D[:, 1, 1] - D[:, 0, 1] * D[:, 1, 0]], 1)], 1)
    return (inv / det[:, None, None]).astype(np.float32)


REST_FAR = np.array([[0.0, 0.0, 0.0], [1.1, 0.1, -0.3], [0.3, 0.9, 0.2], [-0.2, 0.4, 1.3]])   # a generic rest tet
X_FAR, Y_FAR = np.array([1000.5, -2000.25, 500.125]), np.array([-700.25, 300.5, 1200.75])


def single_tet_mesh(F_unit, F_far):
    """Disjoint tets, one component each: unit right tets at rest (B = I exactly) deformed to F_unit with vertex 0 at the
    origin (F exact), and the generic rest tet far from the origin deformed to about F_far there.  Returns verts, tets,
    x, B [T, 3, 3] (fp32) and the F the kernel computes, double(x_k - x_0 in fp32) B in fp64."""
    nu, nf = len(F_unit), len(F_far)
    rest = np.concatenate([np.eye(4, 3, -1)[None] + np.array([4.0 * k, 0.0, 0.0]) for k in range(nu)]
                          + [REST_FAR[None] + X_FAR + np.array([0.0, 4.0 * k, 0.0]) for k in range(nf)]).astype(np.float32)
    tets = np.arange(4 * (nu + nf), dtype=np.int32).reshape(-1, 4)
    xu = np.concatenate([np.zeros((nu, 1, 3)), np.asarray(F_unit).transpose(0, 2, 1)], axis=1)
    Dr = (REST_FAR[1:] - REST_FAR[0]).T
    xf = Y_FAR + np.concatenate([np.zeros((nf, 1, 3)), (np.asarray(F_far) @ Dr).transpose(0, 2, 1)], axis=1)
    x = np.concatenate([xu, xf]).astype(np.float32)                          # [T, 4, 3]
    B = _host_B(rest.reshape(-1, 3), tets)
    E = (x[:, 1:] - x[:, :1]).astype(np.float64)                             # fp32 differences, [T, k, r]
    F = E[:, 0, :, None] * B[:, 0, None, :].astype(np.float64)              # the kernel's sum over k (products exact)
    F = F + E[:, 1, :, None] * B[:, 1, None, :].astype(np.float64)
    F = F + E[:, 2, :, None] * B[:, 2, None, :].astype(np.float64)
    return rest.reshape(-1, 3), tets, x, B, F


def _all_cases(rng, gpu):
    fam = edge_cases(rng, gpu)
    fam["random"] = random_F(rng, 200 if gpu else 2000)
    return fam


def test_apply_reenact_within_bound():
    """psd_apply_kernel's fp32 product against the fp64 projection, per tet and corner: |g - g64|_max <= KAPPA (u
    lambda_max + FLT_MIN) wt |B| |dF|abs|, on the unit right tet and the far generic tet (the bound of the GPU test)."""
    rng = np.random.default_rng(8)
    for name, Fc in _all_cases(rng, False).items():
        _, _, x, B, F = single_tet_mesh(Fc, Fc)
        vs = rng.standard_normal(x.shape).astype(np.float32)
        worst = 0.0
        for order, c3 in ((2, 0.0), (4, C3), (2, C3)):
            kind, _, op32 = project_reenact(F, order, c3 != 0.0)
            act = kind != 0
            P, lmax = eigh_reference(F, kind, order)
            wt = np.where(kind == 1, COEF[1], c3)
            g, _ = apply_reenact({k: v[act] for k, v in op32.items()}, B[act], vs[act], 1.0)
            ref, mag, _ = reference_corners(P[act], B[act], vs[act], 1.0)
            g = g.astype(np.float64) * wt[act, None, None]
            ratio = np.abs(g - wt[act, None, None] * ref).max(axis=(1, 2)) / ((U32 * lmax[act] + FLT_MIN) * mag * wt[act])
            worst = max(worst, ratio.max())
        print(f"apply {name}: worst |g - g64| / (u lambda_max |B| |dF|) = {worst:.3g} (KAPPA {KAPPA})")
        assert worst <= (KAPPA / 4 if name == "random" else KAPPA), name


def test_curvature_floor():
    """q = Dh : D' in fp32 is >= 0 up to A+'s own rounding: q >= -KAPPA_Q u lambda_max |dF|^2, for random dF and for dF
    in the kernel of A+ and of the clamped twist modes, where rounding decides the sign."""
    rng = np.random.default_rng(9)
    worst = 0.0
    for name, F in _all_cases(rng, False).items():
        for order, amips in ((2, False), (4, False), (2, True)):
            kind, op, op32 = project_reenact(F, order, amips)
            act = kind != 0
            if not act.any():
                continue
            o = {k: v[act] for k, v in op.items()}
            _, lmax = eigh_reference(F[act], kind[act], order)
            lam, Q = np.linalg.eigh(o["Ap"])
            z = Q[:, :, 0]                                                    # A+'s smallest eigen-direction
            Dh = np.zeros((act.sum(), 3, 3))
            Dh[:, [0, 1, 2], [0, 1, 2]] = z
            for P, (i, j) in enumerate(PAIRS):                              # the twist mode whose eigenvalue is clamped
                sgn = np.where(o["ls"][:, P] == 0.0, 1.0, -1.0)
                Dh[:, i, j], Dh[:, j, i] = 1.0, sgn
            for dF in (np.einsum("tri,tij,tcj->trc", o["U"], Dh, o["V"]), rng.standard_normal((act.sum(), 3, 3))):
                vs = np.concatenate([np.zeros((len(dF), 1, 3)), dF.transpose(0, 2, 1)], axis=1)
                B = np.broadcast_to(np.eye(3, dtype=np.float32), dF.shape)
                _, q = apply_reenact({k: v[act] for k, v in op32.items()}, B, vs, 1.0)
                dFr = np.asarray(vs, np.float32)[:, 1:].transpose(0, 2, 1).astype(np.float64)
                r = -q.astype(np.float64) / (U32 * lmax * (dFr ** 2).sum(axis=(1, 2)))
                worst = max(worst, r.max())
    print(f"curvature: worst -q / (u lambda_max |dF|^2) = {worst:.3g} (KAPPA_Q {KAPPA_Q})")
    assert worst <= KAPPA_Q


# ---------------------------------------------------------------------------------------------------------------------
# GPU

R_EXACT = [np.eye(3), np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]),       # exact fp32 rotations
           np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]), 1.5 * np.diag([1.0, -1.0, -1.0])]
ZERO_J = [np.array([[1.0, 2.0, 3.0], [4.0, 5.0, 6.0], [0.0, 0.0, 0.0]]), np.zeros((3, 3)),       # flat; a point
          np.array([[1.0, 1.0, 0.5], [0.0, 0.0, 0.0], [2.0, 2.0, 0.0]])]


def single_tet_cases():
    """The single-tet mesh of the GPU tests and its families: unit right tets at the edge cases, exact rotations and J = 0
    exactly; the far generic tet at the edge cases."""
    rng = np.random.default_rng(12)
    fam = _all_cases(rng, True)
    names = [k for k, v in fam.items() for _ in v]
    Fc = np.concatenate(list(fam.values()))
    F_unit = np.concatenate([Fc, f32(np.stack(R_EXACT)), np.stack(ZERO_J)])
    labels = ([f"unit {k}" for k in names] + ["rotation"] * len(R_EXACT) + ["zero J"] * len(ZERO_J)
              + [f"far {k}" for k in names])
    V, T, x, B, F = single_tet_mesh(F_unit, Fc)
    return dict(V=V, T=T, x=x, B=B, F=F, labels=np.array(labels))


@pytest.fixture(scope="module")
def gpu_mesh():
    return single_tet_cases()


def _gpu_run(ext, m, kw):
    from tssplat_b200.newton import DevicePCG
    sp = _handle(ext, m["V"], m["T"], enable_amips=True, **kw)
    return sp, DevicePCG(sp, hessian="psd")


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(), dict(deterministic=True)], ids=["default", "det"])
def test_per_tet_products_against_fp64(ext, gpu_mesh, kw):
    """Every tet's corner product of tsb_pcg_hvp_psd (c1 = 0) against the fp64 eigh projection within the calibrated
    bound, orders 2 and 4, AMIPS off and on; J = 0 tets add exact zeros; the curvature record against fp64 sums."""
    m = gpu_mesh
    sp, ws = _gpu_run(ext, m, kw)
    T = len(m["T"])
    rng = np.random.default_rng(13)
    v_np = rng.standard_normal((4 * T, 3)).astype(np.float32)
    vs = v_np.reshape(T, 4, 3)
    x, v = _cuda(m["x"].reshape(-1, 3)), _cuda(v_np)
    c2 = COEF[1]
    worst = {}
    for order in (2, 4):
        for c3 in (0.0, C3):
            hv, curv = ws.hvp_psd(x, v, 0.0, c2, order, c3=c3)
            got = hv.double().cpu().numpy().reshape(T, 4, 3)
            cv = curv.double().cpu().numpy()
            assert np.isfinite(got).all() and np.isfinite(cv).all()
            kind, _, _ = project_reenact(m["F"], order, c3 != 0.0)
            P, lmax = eigh_reference(m["F"], kind, order)
            wt = np.where(kind == 1, c2, np.where(kind == 2, c3, 0.0))
            ref, mag, dF = reference_corners(P, m["B"], vs, 1.0)
            err = np.abs(got - wt[:, None, None] * ref).max(axis=(1, 2))
            act = kind != 0
            ratio = err[act] / ((U32 * lmax[act] + FLT_MIN) * mag[act] * wt[act])
            for lab in np.unique(m["labels"][act]):
                sel = m["labels"][act] == lab
                worst[lab] = max(worst.get(lab, 0.0), ratio[sel].max())
            bad = np.nonzero(ratio > KAPPA)[0]
            assert not len(bad), (order, c3, [(m["labels"][act][i], ratio[i]) for i in bad[:8]])
            assert (got[~act] == 0.0).all(), (order, c3)                     # inactive tets: exact zeros
            assert (kind[m["labels"] == "zero J"] == 0).all()
            # the record: (vMv = 0 on face-isolated tets, v^T P(H_b) v, v^T P(H_a) v) in fp64
            q = np.einsum("ti,tij,tj->t", dF.reshape(-1, 9), P, dF.reshape(-1, 9))
            dFa = np.einsum("tkr,tkc->trc", np.abs(vs[:, 1:] - vs[:, :1]).astype(np.float64), np.abs(m["B"]).astype(np.float64))
            qt = KAPPA * (U32 * lmax + FLT_MIN) * (dFa ** 2).sum(axis=(1, 2))
            assert cv[1] == 0.0
            for k, K in ((2, 1), (3, 2)):
                ref_q = q[kind == K].sum()
                assert abs(cv[k] - ref_q) <= qt[kind == K].sum() + 2 * U32 * abs(ref_q), (order, c3, k, cv[k], ref_q)
            tot = c2 * q[kind == 1].sum() + c3 * q[kind == 2].sum()
            assert abs(cv[0] - tot) <= c2 * qt[kind == 1].sum() + c3 * qt[kind == 2].sum() + 4 * U32 * abs(tot)
    print(f"{kw}: worst per-tet |hv - hv64| / (u lambda_max wt |B| |dF|) by family (KAPPA {KAPPA}): "
          + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


@pytest.mark.gpu
def test_known_answers_on_single_tets(ext, gpu_mesh):
    """AMIPS at exact rotations is already PSD: the projected product is the exact one (tsb_hvp_ex) on those tets.  An
    inverted tet with AMIPS on gets the barrier term alone: its corners are bitwise those with c3 = 0."""
    m = gpu_mesh
    sp, ws = _gpu_run(ext, m, dict(deterministic=True))
    T = len(m["T"])
    v_np = np.random.default_rng(14).standard_normal((4 * T, 3)).astype(np.float32)
    x, v = _cuda(m["x"].reshape(-1, 3)), _cuda(v_np)
    c2 = COEF[1]
    hp, _ = ws.hvp_psd(x, v, 0.0, c2, 2, c3=C3)
    he, _ = sp.hvp(x, v, 0.0, c2, 2, c3=C3)
    hp, he = hp.double().cpu().numpy().reshape(T, 4, 3), he.double().cpu().numpy().reshape(T, 4, 3)
    rot = m["labels"] == "rotation"
    kind, _, _ = project_reenact(m["F"], 2, True)
    assert (kind[rot] == 2).all()
    _, lmax = eigh_reference(m["F"][rot], kind[rot], 2)
    assert np.allclose(lmax, [4 / 3] * 3 + [4 / 3 / 1.5 ** 2], rtol=1e-12)     # AMIPS is scale-free: H ~ 1 / s^2
    _, mag, _ = reference_corners(np.zeros((rot.sum(), 9, 9)), m["B"][rot], v_np.reshape(T, 4, 3)[rot], C3)
    err = np.abs(hp[rot] - he[rot]).max(axis=(1, 2))
    assert (err <= KAPPA * U32 * lmax * mag).all(), err / (U32 * lmax * mag)
    inv = kind == 1
    assert inv.sum() > 20
    for order in (2, 4):
        h0, _ = ws.hvp_psd(x, v, 0.0, c2, order, c3=0.0)
        h3, _ = ws.hvp_psd(x, v, 0.0, c2, order, c3=C3)
        h0, h3 = h0.cpu().numpy().reshape(T, 4, 3), h3.cpu().numpy().reshape(T, 4, 3)
        assert np.array_equal(h0[inv], h3[inv]), order
        assert (h0[kind == 2] == 0.0).all()                                    # AMIPS off: J > 0 tets are inactive
