"""The fp64 model of the device Newton step and the GPU helpers its test suites share (test_pcg_device, test_newton_*).

The model mirrors the device path: one batched PCG state machine (and its Steihaug-Toint variant inside a radius), the
kernel's 3x3 block preconditioner, two step rules (damped and trust-region, each with the proximal terms), one fp64
reference of the whole step driven by a small step descriptor like tsb_capi.cu's NewtonStep, and one re-enactment of a
device step from the public calls.  Not a test module: the suites import what they use by name."""
import functools
from collections import namedtuple

import numpy as np
import pytest

from tssplat_b200.mesh import connected_components, make_pack, perturb

# solve statuses (tsb_pcg_solve / tsb_pcg_solve_tr) and Newton statuses
MAXITER, CONVERGED, NEGCURV, NEGCURV_FIRST, ZERO_RHS, BOUNDARY, NEGCURV_BOUNDARY = range(7)
ACTIVE, N_CONVERGED, STALLED = 0, 1, 2
CHUNK = 256
ALPHAS = [2.0 ** -k for k in range(8)]
OPTS = dict(max_iter=20, rtol=1e-2, rel_floor=1e-6, tau=1e-3, mu_min=1e-12, mu_max=1e12, gtol=0.0, sigma=1e-4, eta=0.9,
            n_alpha=8)
TR_OPTS = dict(max_iter=20, rtol=1e-2, rel_floor=1e-6, gtol=0.0, radius_init=1.0, radius_min=1e-12, radius_max=1e12,
               accept=1e-4, eta=0.9)
TRLS_OPTS = dict(TR_OPTS, n_alpha=8, sigma=1e-4)
COEF = (2e-4 / 3, 2e-4)
C3 = 1e-4
GPU_SLACK = 8                 # steps the GPU runs on the mixed 64 x 4096 pack may take over the fp64 reference's count
MAX_ROUNDING_FLIPS = 4        # tets one step may newly invert on a sphere through fp32 rounding (test_convergence_mixed_pack)
WEIGHT_SCALES = {"small": 1e-4, "large": 10.0}     # proximal weights, times the sphere's largest Hessian diagonal entry

# Steps the fp64 references need on the small mixed pack (reference_problem) until every sphere they must converge is
# CONVERGED; the GPU runs may take GPU_SLACK more.
# Damped, AMIPS off and on: every sphere.
REF_STEPS = {False: 12, True: 20}
# Proximal, per weight scale.  Under the large weight the rough sphere is held near an anchor with inverted tets: its
# minimiser keeps tets at J ~ 0, where the order-2 barrier's curvature jumps, and the step sizes keep cycling without
# meeting gtol (Phi still falls at every step).
PROX_REF_STEPS = {"small": 12, "large": 2}
# Projected: with w = 0 ("plain") every sphere, the rough one included (the exact reference needs 12); with the small
# weight the two quiet spheres.  There the rough sphere takes the full step every time and Phi falls at every step, but
# the projected model drops the negative curvature of its remaining inverted tets, so the iteration is only linearly
# convergent and does not reach gtol within 20 steps.
PSD_REF_STEPS = {"plain": 7, "small": 2}
PSD_MUST = {"plain": (0, 1, 2), "small": (1, 2)}
# Trust region: plain, AMIPS off and on, and proximal at the two weight scales.  With AMIPS off the rough sphere does not
# converge: its model is good (rho ~ 1), but every full step that follows an accepted one would invert a tet the
# accepted step brought to J ~ 0+, so the rule rejects it and cuts the radius to eta alpha^ |d|_M (about 1/20), while an
# accepted step only doubles it; the radius collapses geometrically.  AMIPS, which grows without bound as J -> 0+, keeps
# tets off J = 0 and the rough sphere converges.  Those spheres must converge: every sphere with AMIPS on, the quiet ones
# otherwise.
TR_REF_STEPS = {"plain": 3, "amips": 13, "small": 3, "large": 2}
TR_MUST_ALL = {"amips"}
# Backtracking trust region.  Unlike the trust-region step's reference, this one converges the rough sphere with AMIPS
# off as well.  With the large proximal weight the rough sphere does not converge here either: the anchor holds it next
# to its inverted start, every full step would invert a tet (eta alpha^ between 0.01 and 0.96), each step is backtracked
# to 2^-k on a boundary solve, so the radius becomes max(2^-k |d|_M, Delta / 4) = 2^-k Delta and still shrinks
# geometrically (to radius_min after 29 steps, then STALLED).  The quiet spheres must converge in every variant.
TRLS_REF_STEPS = {"plain": 5, "amips": 13, "small": 10, "large": 2}
TRLS_MUST_ALL = {"plain", "amips", "small"}
REF_EXTRA = 3                 # steps past the pinned count a reference runs (the fixed point must hold)


def f32(v):
    return float(np.float32(v))


def weight_ok(w):
    return bool(np.isfinite(w) and w >= 0)


# ---------------------------------------------------------------------------------------------------------------------
# the solve and the preconditioner


def batched_pcg_reference(H_blocks, b, P, max_iter, rtol):
    """Truncated PCG on every diagonal block at once, as pcg_init / pcg_curv / pcg_update / pcg_dir run it: all
    components take part in every iteration, a stopped one idles with p = 0.  H_blocks, b, P: per component a dense
    [m, m] matrix, a right-hand side [m] and a preconditioner (dense [m, m], or None).  Returns per component a dict
    (d, status, n_hvp, rel_residual, b_dot_d, d_H_d) and the iterations run."""
    S = len(H_blocks)
    ap = lambda c, r: r.copy() if P[c] is None else P[c] @ r
    st = []
    for c in range(S):
        r = np.array(b[c], np.float64)
        z = ap(c, r)
        bb = float(r @ r)
        active = bb != 0.0
        st.append(dict(r=r, z=z, p=z.copy() if active else np.zeros_like(z), d=np.zeros_like(r), rz=float(r @ z), bb=bb,
                       rr=bb, dHd=0.0, n_hvp=0, status=None if active else ZERO_RHS))
    for it in range(max_iter):
        for c, s in enumerate(st):
            if s["status"] is not None:
                continue
            Hp = H_blocks[c] @ s["p"]
            pHp = float(s["p"] @ Hp)
            s["n_hvp"] = it + 1
            if not pHp > 0.0:
                s["status"] = NEGCURV_FIRST if it == 0 else NEGCURV
                if it == 0:
                    s["d"] = s["z"].copy()
                continue
            a = s["rz"] / pHp
            s["d"] = s["d"] + a * s["p"]
            s["r"] = s["r"] - a * Hp
            s["dHd"] += a * a * pHp
            s["z"] = ap(c, s["r"])
            rz, s["rr"] = float(s["r"] @ s["z"]), float(s["r"] @ s["r"])
            if np.sqrt(s["rr"]) <= rtol * np.sqrt(s["bb"]):
                s["status"] = CONVERGED
            s["p"] = s["z"] + (rz / s["rz"]) * s["p"]
            s["rz"] = rz
    out = []
    for c, s in enumerate(st):
        status = MAXITER if s["status"] is None else s["status"]
        rel = 0.0 if status == ZERO_RHS else 1.0 if status == NEGCURV_FIRST else float(np.sqrt(s["rr"] / s["bb"]))
        out.append(dict(d=s["d"], status=status, n_hvp=s["n_hvp"], rel_residual=rel, b_dot_d=float(np.dot(b[c], s["d"])),
                        d_H_d=s["dHd"]))
    return out


def boundary_tau(pMp, dMp, dMd, D2):
    num = D2 - dMd
    den = dMp + np.sqrt(dMp * dMp + pMp * num)
    return num / den if num > 0.0 and den > 0.0 else 0.0


def batched_steihaug(H_blocks, b, P, radius, max_iter, rtol, history=False):
    """tsb_pcg_solve_tr's state machine in fp64 (batched_pcg_reference plus the radius): per component the M-norm
    recurrences pMp, dMp, dMd of the header, the boundary test on the next iterate, and tau p to the boundary at negative
    curvature or on crossing.  P: dense SPD preconditioners (M = P^-1).  A radius of +inf is the plain state machine.
    Returns per component a dict (d, status, n_hvp, rel_residual, b_dot_d, d_H_d, dMd), and with history the iterates and
    the recurrence's dMd after every step."""
    st = []
    for c in range(len(H_blocks)):
        r = np.array(b[c], np.float64)
        z = P[c] @ r
        bb = float(r @ r)
        active = bb != 0.0
        st.append(dict(r=r, z=z, p=z.copy() if active else np.zeros_like(z), d=np.zeros_like(r), rz=float(r @ z), bb=bb, rr=bb,
                       dHd=0.0, n_hvp=0, status=None if active else ZERO_RHS, pMp=float(r @ z), dMp=0.0, dMd=0.0,
                       hist=[(np.zeros_like(r), 0.0)]))
    for it in range(max_iter):
        for c, s in enumerate(st):
            if s["status"] is not None:
                continue
            Hp = H_blocks[c] @ s["p"]
            pHp = float(s["p"] @ Hp)
            s["n_hvp"] = it + 1
            D = float(radius[c]) if radius[c] > 0 else 0.0
            bst = None
            if np.isfinite(D):
                if not pHp > 0.0:
                    bst = NEGCURV_BOUNDARY
                else:
                    a = s["rz"] / pHp
                    if s["dMd"] + 2.0 * a * s["dMp"] + a * a * s["pMp"] >= D * D:
                        bst = BOUNDARY
            if bst is not None:
                tau = boundary_tau(s["pMp"], s["dMp"], s["dMd"], D * D)
                s["d"] = s["d"] + tau * s["p"]
                s["dHd"] += tau * tau * pHp
                s["dMd"] = s["dMd"] + 2.0 * tau * s["dMp"] + tau * tau * s["pMp"]
                s["status"] = bst
                s["hist"].append((s["d"].copy(), s["dMd"]))
                continue
            if not pHp > 0.0:
                s["status"] = NEGCURV_FIRST if it == 0 else NEGCURV
                if it == 0:
                    s["d"] = s["z"].copy()
                    s["dMd"] = s["pMp"]
                continue
            a = s["rz"] / pHp
            s["d"] = s["d"] + a * s["p"]
            s["r"] = s["r"] - a * Hp
            s["dHd"] += a * a * pHp
            s["dMd"] = s["dMd"] + 2.0 * a * s["dMp"] + a * a * s["pMp"]
            s["hist"].append((s["d"].copy(), s["dMd"]))
            s["z"] = P[c] @ s["r"]
            rz, s["rr"] = float(s["r"] @ s["z"]), float(s["r"] @ s["r"])
            if np.sqrt(s["rr"]) <= rtol * np.sqrt(s["bb"]):
                s["status"] = CONVERGED
            beta = rz / s["rz"]
            s["dMp"] = beta * (s["dMp"] + a * s["pMp"])
            s["pMp"] = rz + beta * beta * s["pMp"]
            s["p"] = s["z"] + beta * s["p"]
            s["rz"] = rz
    out = []
    for c, s in enumerate(st):
        status = MAXITER if s["status"] is None else s["status"]
        rel = 0.0 if status == ZERO_RHS else 1.0 if status == NEGCURV_FIRST else float(np.sqrt(s["rr"] / s["bb"]))
        o = dict(d=s["d"], status=status, n_hvp=s["n_hvp"], rel_residual=rel, b_dot_d=float(np.dot(b[c], s["d"])),
                 d_H_d=s["dHd"], dMd=s["dMd"])
        if history:
            o["hist"] = s["hist"]
        out.append(o)
    return out


def jacobi_inverse_blocks(D, rel_floor, sweeps=8):
    """pcg_blocks_kernel in numpy, operation for operation (fp64): cyclic Jacobi over (0,1), (0,2), (1,2), clamp,
    invert.  D: [n, 3, 3] symmetric.  Returns [n, 6] = (xx, yy, zz, yz, xz, xy)."""
    out = np.zeros((len(D), 6))
    for i, A in enumerate(np.asarray(D, np.float64)):
        a = {(0, 0): A[0, 0], (1, 1): A[1, 1], (2, 2): A[2, 2], (0, 1): A[0, 1], (0, 2): A[0, 2], (1, 2): A[1, 2]}
        V = np.eye(3)
        key = lambda i, j: (min(i, j), max(i, j))
        for _ in range(sweeps):
            if a[(0, 1)] == 0.0 and a[(0, 2)] == 0.0 and a[(1, 2)] == 0.0:
                break
            for p, q in ((0, 1), (0, 2), (1, 2)):
                r = 3 - p - q
                apq = a[(p, q)]
                if apq == 0.0:
                    continue
                with np.errstate(over="ignore"):                     # a tiny a_pq: theta = inf, t = 0, as in the kernel
                    theta = (a[(q, q)] - a[(p, p)]) / (2.0 * apq)
                    t = np.copysign(1.0, theta) / (abs(theta) + np.sqrt(theta * theta + 1.0))
                c = 1.0 / np.sqrt(t * t + 1.0)
                s = t * c
                a[(p, p)] -= t * apq
                a[(q, q)] += t * apq
                a[(p, q)] = 0.0
                apr, aqr = a[key(p, r)], a[key(q, r)]
                a[key(p, r)], a[key(q, r)] = c * apr - s * aqr, s * apr + c * aqr
                vp, vq = V[:, p].copy(), V[:, q].copy()
                V[:, p], V[:, q] = c * vp - s * vq, s * vp + c * vq
        lam = np.array([a[(0, 0)], a[(1, 1)], a[(2, 2)]])
        lmax = lam.max()
        if lmax > 0.0:
            inv = 1.0 / np.maximum(lam, rel_floor * lmax)
            M = (V * inv) @ V.T
            out[i] = [M[0, 0], M[1, 1], M[2, 2], M[1, 2], M[0, 2], M[0, 1]]
    return out


def block_preconditioner(D, shift, rel_floor):
    """The dense block-diagonal preconditioner the kernel builds from the diagonal blocks D [m, 3, 3] plus shift I."""
    inv = jacobi_inverse_blocks(D + float(shift) * np.eye(3), rel_floor)
    B = np.zeros((3 * len(D), 3 * len(D)))
    for i, q in enumerate(inv):
        B[3 * i:3 * i + 3, 3 * i:3 * i + 3] = [[q[0], q[5], q[4]], [q[5], q[1], q[3]], [q[4], q[3], q[2]]]
    return B


def sym6(P):
    """[n, 3, 3] symmetric -> [n, 6] = (xx, yy, zz, yz, xz, xy)."""
    P = np.asarray(P)
    return np.stack([P[:, 0, 0], P[:, 1, 1], P[:, 2, 2], P[:, 1, 2], P[:, 0, 2], P[:, 0, 1]], axis=1)


def planes_of(D):
    D = np.asarray(D)
    return np.stack([np.stack([D[:, 0, 0], D[:, 1, 1], D[:, 2, 2]], 1), np.stack([D[:, 1, 2], D[:, 0, 2], D[:, 0, 1]], 1)])


def _spd(rng, m, lo=0.5, hi=20.0):
    Q = np.linalg.qr(rng.normal(size=(m, m)))[0]
    return (Q * rng.uniform(lo, hi, size=m)) @ Q.T


def _shuffled_mesh():
    """tests/test_hvp.py's "shuffled" mesh: a 3 x 1024 pack relabelled into a larger id space (500 orphans)."""
    pk = make_pack(3, 1024, seed=1)
    rng = np.random.default_rng(8)
    n = len(pk.verts) + 500
    ids = rng.permutation(n)[:len(pk.verts)]
    V = rng.normal(size=(n, 3)).astype(np.float32)
    V[ids] = pk.verts
    T = ids[pk.tets].astype(np.int32)
    x = V.copy()
    x[ids] = perturb(pk, sigma_rel=0.02, seed=1)
    return V, T, x


# ---------------------------------------------------------------------------------------------------------------------
# the two step rules


def new_state(S):
    """Per-sphere rule state: the damping (mu, nu) of the damped rule, the radius of the trust-region rule."""
    return [dict(mu=None, nu=None, radius=None, status=ACTIVE) for _ in range(S)]


def init_shift(st, maxD, o, w=None):
    """mu_c = tau (max (D_v)_ii + w_c) on a sphere's first step, clamped to [mu_min, mu_max]; returns the fp32 shifts
    mu_c + w_c of the solve (w_c read as 0 where it is unusable, and 0 without weights)."""
    out = []
    for s, m, wc in zip(st, maxD, np.zeros(len(st)) if w is None else w):
        we = float(np.float32(wc)) if weight_ok(wc) else 0.0
        if s["mu"] is None:
            s["mu"] = min(f32(o["mu_max"]), max(f32(o["mu_min"]), f32(o["tau"]) * (float(m) + we)))
            s["nu"] = 2.0
        out.append(s["mu"] + we)
    return np.array(out, np.float32)


def decide_damped(s, g, bd, dHd, mu_f, dd, dE, ahat, o, w=0.0, dx=0.0, alphas=ALPHAS):
    """newton_decide_kernel<PROX> for one sphere, operation for operation in fp64: updates the state s (mu, nu, status)
    and returns (alpha, k, dPhi of the step, rho).  bd and dHd are the solve's fp32 records, mu_f the fp32 shift the
    solve used, dd = d.d, dE[k] = E(x + alpha_k d) - E(x) and ahat the inversion-free step over (0, 1], fp32.  With a
    weight w > 0, dPhi_k = dE_k + w (a_k dx + a_k^2 dd / 2) with dx = d.(x - y) in place of dE_k, and pred uses
    mu' = mu_f - w; an unusable w freezes the sphere as STALLED."""
    if s["status"] != ACTIVE:
        return 0.0, -1, 0.0, 0.0
    if not weight_ok(w):
        s["status"] = STALLED
        return 0.0, -1, 0.0, 0.0
    if g <= f32(o["gtol"]):
        s["status"] = N_CONVERGED
        return 0.0, -1, 0.0, 0.0
    w = float(np.float32(w))
    dphi = [float(dE[k]) + w * (a * dx + 0.5 * a * a * dd) if w > 0 else float(dE[k]) for k, a in enumerate(alphas[:o["n_alpha"]])]
    lim = f32(o["eta"]) * float(ahat)
    ks = -1
    if bd > 0.0:
        for k in range(o["n_alpha"]):
            a = alphas[k]
            if a < lim and dphi[k] <= -f32(o["sigma"]) * a * bd:
                ks = k
                break
    pred = bd - 0.5 * (dHd - (float(mu_f) - w) * dd)
    rho = -dphi[0] / pred if pred > 0.0 else 1.0
    if ks == 0:
        t = 2.0 * rho - 1.0
        s["mu"] = max(f32(o["mu_min"]), s["mu"] * max(1.0 / 3.0, 1.0 - t * t * t))
        s["nu"] = 2.0
    else:
        s["mu"] = min(f32(o["mu_max"]), s["mu"] * s["nu"])
        s["nu"] *= 2.0
    if ks < 0 and s["mu"] == f32(o["mu_max"]):
        s["status"] = STALLED
    return (alphas[ks], ks, dphi[ks], rho) if ks >= 0 else (0.0, -1, 0.0, rho)


def init_radius(st, bPb, o):
    """Delta_c = clamp(radius_init sqrt(b^T P b), radius_min, radius_max) on a sphere's first step; the fp32 radii."""
    for s, q in zip(st, bPb):
        if s["radius"] is None:
            s["radius"] = min(f32(o["radius_max"]), max(f32(o["radius_min"]), f32(o["radius_init"]) * float(np.sqrt(q))))
    return np.array([s["radius"] for s in st], np.float32)


def decide_tr(s, g, bd, dHd, dMd, pcg_status, dphi, ahat, o, w=0.0):
    """newton_decide_tr_kernel<PROX, LS> for one sphere in fp64; s = dict(radius, status), updated.  bd, dHd: the
    solve's records (fp32), dMd = |d|_M^2, dphi[k] = Phi(x + 2^-k d) - Phi(x), ahat the inversion-free step.  With
    o["n_alpha"] > 1 (backtracking, a non-null tsb_newton_backtrack_t), a step the trust-region rule rejects is
    backtracked to the largest 2^-k (k >= 1) below eta alpha^ with the Armijo decrease, and the radius then becomes
    max(2^-k |d|_M, Delta / 4), clamped; without it only dphi[0] is read.  Returns (alpha, rho, pred, delta)."""
    if s["status"] != ACTIVE:
        return 0.0, 0.0, 0.0, 0.0
    if not weight_ok(w):
        s["status"] = STALLED
        return 0.0, 0.0, 0.0, 0.0
    if g <= f32(o["gtol"]):
        s["status"] = N_CONVERGED
        return 0.0, 0.0, 0.0, 0.0
    pred = bd - 0.5 * dHd
    rho = -dphi[0] / pred if pred > 0.0 else 0.0
    dn = float(np.sqrt(dMd))
    lim = f32(o["eta"]) * float(ahat)
    flips = not (1.0 < lim)
    old = s["radius"]
    if flips:
        new = min(0.25 * old, lim * dn)
    elif not rho >= 0.25:
        new = 0.25 * dn
    elif rho > 0.75 and pcg_status in (BOUNDARY, NEGCURV_BOUNDARY):
        new = min(2.0 * old, f32(o["radius_max"]))
    else:
        new = old
    if not flips and pred > 0.0 and rho > f32(o["accept"]):
        s["radius"] = new
        return 1.0, rho, pred, dphi[0]
    if bd > 0.0:
        for k in range(1, int(o.get("n_alpha", 1))):
            a = ALPHAS[k]
            if a < lim and dphi[k] <= -f32(o["sigma"]) * a * bd:
                s["radius"] = min(f32(o["radius_max"]), max(f32(o["radius_min"]), max(a * dn, 0.25 * old)))
                return a, rho, pred, dphi[k]
    s["radius"] = new
    if new < f32(o["radius_min"]):
        s["status"] = STALLED
    return 0.0, rho, pred, 0.0


# ---------------------------------------------------------------------------------------------------------------------
# the fp64 problem and the fp64 reference of the step


def tet_hessians(orc, x, order, c3, project):
    """[T, 9, 9] weighted F-space Hessians c2-free: barrier on J < 0 tets, c3 AMIPS on J > 0 ones (projected or not)."""
    from test_hess_diag import psi_hessians
    F = (orc.G @ np.asarray(x, np.float64).reshape(-1)).reshape(-1, 3, 3)
    Hb = psi_hessians(F, order=order)
    Ha = psi_hessians(F, amips=True) if c3 else np.zeros_like(Hb)
    if project:
        w, Q = np.linalg.eigh(0.5 * (Hb + Hb.transpose(0, 2, 1)))
        Hb = np.einsum("tij,tj,tkj->tik", Q, np.maximum(w, 0), Q)
        if c3:
            w, Q = np.linalg.eigh(0.5 * (Ha + Ha.transpose(0, 2, 1)))
            Ha = np.einsum("tij,tj,tkj->tik", Q, np.maximum(w, 0), Q)
    return Hb, Ha


def dense_sphere_hessians(orc, pk, x, c1, c2, c3, order, project):
    """Dense per-sphere c1 M + c2 sum K^T H_b K + c3 sum K^T H_a K (exact or projected tet blocks)."""
    from test_hess_diag import corner_G
    Hb, Ha = tet_hessians(orc, x, order, c3, project)
    Ht = c2 * Hb + c3 * Ha
    Gk = corner_G(orc).transpose(0, 2, 1, 3).reshape(orc.nele, 9, 12)          # [T, 9, 4 corners x 3]
    K = np.einsum("tma,tmn,tnb->tab", Gk, Ht, Gk)
    M = orc.M.toarray()
    out = []
    for s in range(pk.num_spheres):
        v0, v1 = pk.vert_offsets[s], pk.vert_offsets[s + 1]
        H = c1 * M[3 * v0:3 * v1, 3 * v0:3 * v1]
        for t in np.nonzero((orc.tets[:, 0] >= v0) & (orc.tets[:, 0] < v1))[0]:
            idx = np.concatenate([3 * (orc.tets[t, k] - v0) + np.arange(3) for k in range(4)])
            H[np.ix_(idx, idx)] += K[t]
        out.append(H)
    return out


class Fp64Problem:
    """Per-sphere fp64 energy, gradient, dense Hessian blocks, line search and inversion bound of a pack, from
    ReferenceEnergyOracle and the matrix-form HVPs of test_hvp / test_hvp_amips."""

    def __init__(self, pk, c1, c2, c3, order=2):
        from oracle.tet_energy_oracle import ReferenceEnergyOracle
        self.pk, self.orc = pk, ReferenceEnergyOracle(pk.verts, pk.tets)
        self.c1, self.c2, self.c3, self.order = c1, c2, c3, order
        self.vo, self.S = pk.vert_offsets, pk.num_spheres
        self.tsid = np.searchsorted(self.vo, pk.tets[:, 0], side="right") - 1

    def sphere_energy(self, x):
        from oracle.tet_energy_oracle import _det3
        x = np.asarray(x, np.float64).reshape(-1)
        Mx = self.orc.M @ x
        F = (self.orc.G @ x).reshape(-1, 3, 3)
        J = _det3(F)
        bar = np.maximum(-J, 0) ** self.order
        ok = J > 0
        tr = (F * F).sum(axis=(1, 2))
        psi = np.where(ok, tr / (3.0 * np.where(ok, J, 1.0) ** (2.0 / 3.0)) - 1.0, 0.0)
        sm = 0.5 * (x * Mx).reshape(-1, 3).sum(1)
        E = np.array([self.c1 * sm[self.vo[s]:self.vo[s + 1]].sum() for s in range(self.S)])
        E += np.bincount(self.tsid, self.c2 * bar + self.c3 * psi, minlength=self.S)
        return E, np.bincount(self.tsid, J < 0, minlength=self.S).astype(int)

    def objective(self, x, y=None, w=None):
        """Per-sphere Phi_c = E_c + (w_c / 2) |x_c - y_c|^2 (E_c without an anchor)."""
        E, _ = self.sphere_energy(x)
        if w is None:
            return E
        r = (np.asarray(x, np.float64) - y).reshape(-1, 3)
        return E + 0.5 * w * np.array([(r[self.vo[s]:self.vo[s + 1]] ** 2).sum() for s in range(self.S)])

    def grad(self, x):
        g = self.orc.backward(1.0, x, self.c1, self.c2, self.order)
        if self.c3:
            g = g + self.orc.amips_backward(1.0, x, self.c3)
        return g.reshape(-1)

    def hess_blocks(self, x, project=False):
        """Dense H_c per sphere.  Exact: spheres share no vertices, so one HVP along the sum of every sphere's j-th unit
        vector gives column j of every block.  project: assembled from the PSD-projected tet Hessians."""
        if project:
            return dense_sphere_hessians(self.orc, self.pk, x, self.c1, self.c2, self.c3, self.order, True)
        from test_hvp import hvp
        from test_hvp_amips import amips_hvp_terms
        m3 = 3 * np.diff(self.vo)
        H = [np.zeros((k, k)) for k in m3]
        for j in range(int(m3.max())):
            e = np.zeros(3 * len(self.pk.verts))
            for s in range(self.S):
                if j < m3[s]:
                    e[3 * self.vo[s] + j] = 1.0
            col = hvp(self.orc, x, e, self.c1, self.c2, self.order).reshape(-1)
            if self.c3:
                col = col + self.c3 * amips_hvp_terms(self.orc, x, e)[0]
            for s in range(self.S):
                if j < m3[s]:
                    H[s][:, j] = col[3 * self.vo[s]:3 * self.vo[s + 1]]
        return H

    def inversion_bound(self, x, d):
        from test_line_search import cubic_coeffs, first_root
        r = first_root(cubic_coeffs(self.orc, x, d), 1.0)
        out = np.full(self.S, np.inf)
        np.minimum.at(out, self.tsid, r)
        return out


# What differs between the device's Newton steps (tsb_capi.cu's NewtonStep): the rule ("damped" or "tr"), whether a
# rejected step is backtracked along 2^-k (the damped rule always searches its step sizes), and whether the solve
# multiplies by the projected Hessian H+ (the preconditioner keeps the exact diagonal blocks).
Step = namedtuple("Step", "kind backtrack projected")
STEPS = {"lm": Step("damped", True, False), "prox": Step("damped", True, False), "psd": Step("damped", True, True),
         "tr": Step("tr", False, False), "trls": Step("tr", True, False)}


def reference(P, x0, n_steps, o, step, y=None, w=None):
    """The device Newton step's algorithm in fp64: -grad, frozen spheres zeroed, the proximal pull (with an anchor y and
    weights w), the diagonal blocks, the kernel's preconditioner on D + shift I (shift mu + w for the damped rule, w for
    the trust-region rule), the batched solve on H + shift I (PCG, or Steihaug-Toint inside the radius), the energy
    changes at the step sizes from the oracle's energies, its inversion cubic, the rule, the step.  Returns the final x
    and per step and sphere a dict of what the rule saw and decided."""
    x = np.asarray(x0, np.float64).reshape(-1).copy()
    prox = y is not None
    y = np.asarray(y, np.float64).reshape(-1) if prox else None
    w = np.asarray(w, np.float64) if prox else np.zeros(P.S)
    damped = step.kind == "damped"
    alphas = ALPHAS[:o["n_alpha"] if step.backtrack else 1]
    st = new_state(P.S)
    sl = [slice(3 * P.vo[s], 3 * P.vo[s + 1]) for s in range(P.S)]
    hist = []
    for _ in range(n_steps):
        b = -P.grad(x)
        for s in range(P.S):
            if st[s]["status"] != ACTIVE or not weight_ok(w[s]):
                b[sl[s]] = 0.0
            elif w[s]:
                b[sl[s]] -= w[s] * (x[sl[s]] - y[sl[s]])
        He = dense_sphere_hessians(P.orc, P.pk, x, P.c1, P.c2, P.c3, P.order, False) if step.projected else P.hess_blocks(x)
        H = P.hess_blocks(x, project=True) if step.projected else He
        D = [np.stack([Hc[3 * i:3 * i + 3, 3 * i:3 * i + 3] for i in range(len(Hc) // 3)]) for Hc in He]
        shift = init_shift(st, [Dc[:, [0, 1, 2], [0, 1, 2]].max() for Dc in D], o, w) if damped else w
        Pc = [block_preconditioner(Dc, m, o["rel_floor"]) for Dc, m in zip(D, shift)]
        A = [Hc + float(m) * np.eye(len(Hc)) for Hc, m in zip(H, shift)]
        bs = [b[sl[s]] for s in range(P.S)]
        if damped:
            sol = batched_pcg_reference(A, bs, Pc, o["max_iter"], o["rtol"])
        else:
            rad_in = init_radius(st, [float(q @ Pq @ q) for q, Pq in zip(bs, Pc)], o)
            sol = batched_steihaug(A, bs, Pc, rad_in, o["max_iter"], o["rtol"])
        d = np.concatenate([r["d"] for r in sol])
        E0, inv0 = P.sphere_energy(x)
        dE = np.stack([P.sphere_energy(x + a * d)[0] - E0 for a in alphas], axis=1)
        ahat = P.inversion_bound(x, d)
        out = []
        for s, r in enumerate(sol):
            ds = r["d"]
            dd = float(ds @ ds)
            dx = float(ds @ (x[sl[s]] - y[sl[s]])) if w[s] > 0 else 0.0
            h = dict(g=float(np.linalg.norm(bs[s])), pcg=r["status"], bd=r["b_dot_d"], dHd=r["d_H_d"], dd=dd, E0=E0[s],
                     inv0=inv0[s], ahat=float(ahat[s]),
                     phi0=E0[s] + (0.5 * w[s] * float((x[sl[s]] - y[sl[s]]) @ (x[sl[s]] - y[sl[s]])) if prox else 0.0))
            if damped:
                h.update(zip(("alpha", "k", "delta", "rho"),
                             decide_damped(st[s], h["g"], h["bd"], h["dHd"], shift[s], dd, dE[s], ahat[s], o, w[s], dx)),
                         mu=st[s]["mu"], mu_f=float(shift[s]))
            else:
                dphi = [dE[s, k] + (w[s] * (a * dx + 0.5 * a * a * dd) if w[s] > 0 else 0.0) for k, a in enumerate(alphas)]
                h.update(radius_in=st[s]["radius"], dphi=dphi)
                h.update(zip(("alpha", "rho", "pred", "delta"),
                             decide_tr(st[s], h["g"], h["bd"], h["dHd"], r["dMd"], r["status"], dphi, ahat[s], o, w[s])),
                         radius=st[s]["radius"])
            h["status"] = st[s]["status"]
            out.append(h)
        for s in range(P.S):
            x[sl[s]] += out[s]["alpha"] * sol[s]["d"]
        hist.append(out)
    return x, hist


@functools.lru_cache(maxsize=None)
def reference_problem(amips=False, round32=True, scale=None, method="lm"):
    """The small mixed pack the fp64 references run on: make_pack(3, 256) at 0.02 h with sphere 0 at 0.35 h (inverted
    tets), started at x0 (rounded to fp32 with round32), AMIPS on or off.  Returns (P, x0, w, o): the proximal weights
    w_c = WEIGHT_SCALES[scale] times the sphere's largest Hessian diagonal entry at the start (None without a scale),
    and the method's options with gtol = 1e-3 times the smallest starting |g_c|."""
    pk = make_pack(3, 256, seed=4)
    x = perturb(pk, sigma_rel=0.02, seed=1).astype(np.float64)
    rough = perturb(pk, sigma_rel=0.35, seed=3)
    x[pk.vert_offsets[0]:pk.vert_offsets[1]] = rough[pk.vert_offsets[0]:pk.vert_offsets[1]]
    if round32:
        x = x.astype(np.float32).astype(np.float64)
    P = Fp64Problem(pk, *COEF, C3 if amips else 0.0)
    w = None
    if scale is not None:
        w = np.array([np.float32(WEIGHT_SCALES[scale] * np.diag(Hc).max()) for Hc in P.hess_blocks(x.reshape(-1))], np.float64)
    g0 = [np.linalg.norm(P.grad(x)[3 * P.vo[s]:3 * P.vo[s + 1]]) for s in range(P.S)]
    o = dict({"tr": TR_OPTS, "trls": TRLS_OPTS}.get(method, OPTS), gtol=1e-3 * min(g0))
    return P, x, w, o


# The fp64 reference runs: method and variant -> (reference_problem's amips, round32 and scale; steps run; spheres that
# must converge; the pinned step count they must converge within).  "amips-off" / "amips-on" and "plain" / "amips"
# minimise E, "small" and "large" the proximal objective anchored at the start.
REFERENCE_RUNS = {
    ("lm", "amips-off"): ((False, False, None), REF_STEPS[False] + REF_EXTRA, (0, 1, 2), REF_STEPS[False]),
    ("lm", "amips-on"): ((True, False, None), REF_STEPS[True] + REF_EXTRA, (0, 1, 2), REF_STEPS[True]),
    ("prox", "small"): ((False, True, "small"), PROX_REF_STEPS["small"] + REF_EXTRA, (0, 1, 2), PROX_REF_STEPS["small"]),
    ("prox", "large"): ((False, True, "large"), PROX_REF_STEPS["small"] + REF_EXTRA, (1, 2), PROX_REF_STEPS["large"]),
    ("psd", "plain"): ((False, True, None), 20, PSD_MUST["plain"], PSD_REF_STEPS["plain"]),
    ("psd", "small"): ((False, True, "small"), 20, PSD_MUST["small"], PSD_REF_STEPS["small"]),
}
for _m, _steps, _all in (("tr", TR_REF_STEPS, TR_MUST_ALL), ("trls", TRLS_REF_STEPS, TRLS_MUST_ALL)):
    for _k in ("plain", "amips", "small", "large"):
        REFERENCE_RUNS[_m, _k] = ((_k == "amips", True, _k if _k in WEIGHT_SCALES else None), _steps[_k] + REF_EXTRA,
                                  (0, 1, 2) if _k in _all else (1, 2), _steps[_k])


@functools.lru_cache(maxsize=None)
def reference_run(method, variant):
    """(P, x0, w, o, must, pinned, x, hist) of one fp64 reference run of REFERENCE_RUNS, anchored at x0 with weights."""
    (amips, round32, scale), n, must, pinned = REFERENCE_RUNS[method, variant]
    P, x0, w, o = reference_problem(amips, round32, scale, method if method in ("tr", "trls") else "lm")
    x, hist = reference(P, x0, n, o, STEPS[method], y=None if w is None else x0, w=w)
    return P, x0, w, o, must, pinned, x, hist


def converged_at(hist, S):
    return [next((t for t, step in enumerate(hist) if step[s]["status"] == N_CONVERGED), None) for s in range(S)]


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers


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


def _cuda(a):
    return _torch().from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


_PACKS = {}


def _pack(name):
    """(pack, x): "big" = 64 x 4096 near rest (0.02 h); "mixed" = the same pack with every fourth sphere at 0.35 h;
    "small" = make_pack(3, 512) with sphere 0 at 0.35 h."""
    if name not in _PACKS:
        pk = make_pack(3, 512, seed=4) if name == "small" else make_pack(64, 4096, seed=0, unique=8)
        x = perturb(pk, sigma_rel=0.02, seed=1)
        if name != "big":
            rough = perturb(pk, sigma_rel=0.35, seed=3)
            for s in range(0, pk.num_spheres, 4):
                x[pk.vert_offsets[s]:pk.vert_offsets[s + 1]] = rough[pk.vert_offsets[s]:pk.vert_offsets[s + 1]]
        _PACKS[name] = (pk, x)
    return _PACKS[name]


def _labels(V, T):
    """(sphere id per vertex, 0 on orphans; orphan mask; S)."""
    lab = connected_components(len(V), T)
    used = np.zeros(len(V), bool)
    used[np.unique(T)] = True
    return np.where(used, np.searchsorted(np.unique(lab[used]), lab), 0), ~used, len(np.unique(lab[used]))


def _seg_sum(torch, v, sid, S):
    return torch.zeros(S, dtype=torch.float64, device=v.device).index_add_(0, sid, v)


def _sphere_max_diag(torch, planes, sid, orph, S):
    m = planes[0].max(dim=1).values.masked_fill(orph, -np.inf)
    return torch.full((S,), -np.inf, dtype=torch.float32, device=m.device).scatter_reduce_(0, sid, m, "amax")


def _weights(torch, planes, sid, orph, S, scales):
    """w_c = scales[c % len(scales)] times the sphere's largest diagonal entry, float32 [S]."""
    mx = _sphere_max_diag(torch, planes, sid, orph, S)
    sc = torch.tensor(scales, dtype=torch.float32, device="cuda").repeat(S // len(scales) + 1)[:S]
    return (mx * sc).contiguous()


def _records(torch, recs):
    """Every field of every step's record as raw bits in one int32 tensor."""
    return torch.cat([torch.cat([f.reshape(-1).contiguous().view(torch.int32) for f in r]) for r in recs])


def _m_norm(torch, d, inv, sid, orph, S):
    """|d_c|_M per sphere in fp64, M = P^-1 from the [n, 6] inverse blocks (vertices with a zero block carry d = 0)."""
    q = inv.double()
    B = torch.stack([torch.stack([q[:, 0], q[:, 5], q[:, 4]], 1), torch.stack([q[:, 5], q[:, 1], q[:, 3]], 1),
                     torch.stack([q[:, 4], q[:, 3], q[:, 2]], 1)], 1)
    live = (q.abs().sum(1) > 0) & ~orph
    dd = d.double()
    sol = torch.zeros_like(dd)
    sol[live] = torch.linalg.solve(B[live], dd[live].unsqueeze(-1)).squeeze(-1)
    assert not dd[~live].any()
    return _seg_sum(torch, (dd * sol).sum(1)[~orph], sid[~orph], S).sqrt()


def _p_apply(inv, v):
    """P v per vertex in fp64 from the [n, 6] inverse blocks (xx, yy, zz, yz, xz, xy)."""
    q = inv.double()
    return _torch().stack([q[:, 0] * v[:, 0] + q[:, 5] * v[:, 1] + q[:, 4] * v[:, 2],
                           q[:, 5] * v[:, 0] + q[:, 1] * v[:, 1] + q[:, 3] * v[:, 2],
                           q[:, 4] * v[:, 0] + q[:, 3] * v[:, 1] + q[:, 2] * v[:, 2]], 1)


def compose(torch, sp, ws, x, st, c1, c2, c3, o, step, sid, orph, S, y=None, w=None, radius_after=None):
    """One device Newton step of kind step.kind re-enacted from the public calls (energy_grad, hess_diag, set_blocks,
    solve, line_search, axpy) and the numpy rule; st is the per-sphere rule state, updated.  The solve runs on ws, so a
    projected workspace gives the projected step.  For the trust-region rule, after the first step the radius a sphere
    enters the solve with is the step's own record of the previous step (radius_after): the rule's |d|_M comes from d
    and the blocks, the kernel's from its recurrences, and the two differ in the last bits.  Returns the new x and per
    sphere a dict of the rule's inputs and outputs."""
    _, b = sp.energy_grad(x, c1, c2, 2, -1.0, c3=c3)
    keep = ~orph
    wn = w.cpu().numpy() if w is not None else np.zeros(S)
    ok = torch.tensor([s["status"] == ACTIVE and weight_ok(v) for s, v in zip(st, wn)], device="cuda")
    b = torch.where(~ok[sid][:, None] & keep[:, None], torch.zeros_like(b), b)
    if y is not None:
        pull = ok[sid] & keep & (w[sid] != 0)
        b = torch.where(pull[:, None], b + (-w)[sid][:, None] * (x - y), b)
    planes = sp.hess_diag(x, c1, c2, 2, c3=c3)
    if step.kind == "damped":
        shift = torch.from_numpy(init_shift(st, _sphere_max_diag(torch, planes, sid, orph, S).cpu().numpy(), o, wn)).cuda()
        ws.set_blocks(planes, rel_floor=o["rel_floor"], shift=shift)
        res = ws.solve(x, b, c1, c2, 2, c3=c3, max_iter=o["max_iter"], rtol=o["rtol"], shift=shift)
    else:
        inv = ws.set_blocks(planes, rel_floor=o["rel_floor"], shift=w, want_inverse=True)
        bd_ = b.double()
        bPb = _seg_sum(torch, (bd_ * _p_apply(inv, bd_)).sum(1)[keep], sid[keep], S).cpu().numpy()
        if radius_after is not None:
            for s, r in zip(st, radius_after):
                s["radius"] = float(r)
        rad = torch.from_numpy(init_radius(st, bPb, o)).cuda()
        res = ws.solve(x, b, c1, c2, 2, c3=c3, max_iter=o["max_iter"], rtol=o["rtol"], shift=w, radius=rad)
        dMd = (_m_norm(torch, res.d, inv, sid, orph, S) ** 2).cpu().numpy()
    alphas = ALPHAS[:o.get("n_alpha", 1) if step.backtrack else 1]
    ls = sp.line_search(x, res.d, alphas, c1, c2, 2, c3=c3, per_sphere=True)
    gn = _seg_sum(torch, (b.double() ** 2).sum(1)[keep], sid[keep], S).sqrt().cpu().numpy()
    dd = _seg_sum(torch, (res.d.double() ** 2).sum(1)[keep], sid[keep], S).cpu().numpy()
    dx = _seg_sum(torch, (res.d.double() * (x.double() - y.double())).sum(1)[keep], sid[keep], S).cpu().numpy() if y is not None else dd * 0
    bd, dHd, sd, ss, ps = (t.cpu().numpy() for t in (res.b_dot_d, res.d_H_d, ls.sphere_delta[:, :, 0], ls.sphere_max_step, res.status))
    out = []
    for c in range(S):
        h = dict(bd=float(bd[c]), ahat=float(ss[c]))
        if step.kind == "damped":
            h.update(zip(("alpha", "k", "delta", "rho"), decide_damped(st[c], float(gn[c]), float(bd[c]), float(dHd[c]),
                                                                       shift[c].item(), float(dd[c]), sd[c], ss[c], o, wn[c], float(dx[c]))))
        else:
            wc = float(wn[c]) if weight_ok(wn[c]) else 0.0
            h["dphi"] = [float(sd[c, k]) + (wc * (a * dx[c] + 0.5 * a * a * dd[c]) if wc > 0 else 0.0) for k, a in enumerate(alphas)]
            h.update(zip(("alpha", "rho", "pred", "delta"), decide_tr(st[c], float(gn[c]), float(bd[c]), float(dHd[c]), float(dMd[c]),
                                                                      int(ps[c]), h["dphi"], ss[c], o, wn[c])), dMd=float(dMd[c]))
        out.append(h)
    a = torch.tensor([h["alpha"] for h in out], dtype=torch.float32, device="cuda")
    return ws.axpy(x, a, res.d), out


# ---------------------------------------------------------------------------------------------------------------------
# PSD helpers


def _rot(rng):
    Q, R = np.linalg.qr(rng.standard_normal((3, 3)))
    Q = Q * np.sign(np.diag(R))
    return Q if np.linalg.det(Q) > 0 else -Q


def _cases(rng):
    """(name, F): random, rotations and identity, two equal s, near rest, s_3 -> 0-, s_3 ~ -s_2, reflections."""
    out = []
    for k in range(4):
        F = rng.standard_normal((3, 3))
        out.append((f"random{k}", F))
    R = _rot(rng)
    out += [("identity", np.eye(3)), ("rotation", R), ("scaled rotation", 1.7 * R),
            ("two equal", _rot(rng) @ np.diag([1.3, 0.8, 0.8]) @ _rot(rng).T),
            ("near rest", np.eye(3) + 1e-4 * rng.standard_normal((3, 3))),
            ("near rest rotated", R @ (np.eye(3) + 1e-4 * rng.standard_normal((3, 3))))]
    refl = np.diag([1.0, 1.0, -1.0])
    out += [("s3 -> 0-", _rot(rng) @ np.diag([1.2, 0.9, -1e-6]) @ _rot(rng).T),
            ("s3 ~ -s2", _rot(rng) @ np.diag([1.1, 0.7, -0.7 + 1e-9]) @ _rot(rng).T),
            ("reflection", R @ refl), ("reflected stretch", _rot(rng) @ np.diag([1.4, 0.75, -1.0]) @ _rot(rng).T)]
    return out


def _small_mixed():
    """The fp64 references' small mixed pack, rounded to fp32: 3 x 256, sphere 0 at 0.35 h (with inverted tets)."""
    P, x, _, _ = reference_problem()
    return P.pk, x


def _psd_pack(name):
    """(pack, x): "mixed8" = 8 x 1024 with spheres 0 and 4 at 0.35 h; "mixed64" = the mixed 64 x 4096 pack."""
    if name == "mixed64":
        return _pack("mixed")
    pk = make_pack(8, 1024, seed=2)
    x = perturb(pk, sigma_rel=0.02, seed=1)
    rough = perturb(pk, sigma_rel=0.35, seed=3)
    for s in (0, 4):
        x[pk.vert_offsets[s]:pk.vert_offsets[s + 1]] = rough[pk.vert_offsets[s]:pk.vert_offsets[s + 1]]
    return pk, x
