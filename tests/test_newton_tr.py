"""The trust-region Newton step: tsb_pcg_solve_tr (Steihaug-Toint CG inside a per-sphere radius in the preconditioner
norm), tsb_newton_tr_step, DevicePCG.solve(radius=), DeviceNewton.tr_step / minimize(method="tr") and
SmoothnessBarrierEnergy with FLAGS.newton_method = "tr".

CPU: a batched fp64 Steihaug-Toint state machine against dense per-sphere problems (SPD and indefinite): its M-norm
recurrences against the directly computed |d_k|_M, monotone growth, the boundary step, the Cauchy decrease, and the
infinite radius as the plain PCG reference; the step's decision rule with known answers; an fp64 trust-region reference
on the small mixed pack, plain and proximal, which pins the step counts the GPU runs are allowed and whose fixed points
are checked for stationarity (and, proximal, against scipy's trust-region Newton-CG).  GPU: radius +inf is
tsb_pcg_solve_ex bitwise; finite radii are respected in the M-norm and negative curvature is followed to the boundary;
one step against the public calls composed with the numpy rule; determinism, graph replays and independence; handle
variants, orphans and the projected Hessian; convergence on the mixed 64 x 4096 pack; bookkeeping and argument errors;
the module route."""
import ctypes as C

import numpy as np
import pytest

# ext: test_newton_lm's module-scoped fixture, requested by name
from test_newton_lm import (ACTIVE, C3, COEF, GPU_SLACK, MAX_ROUNDING_FLIPS, N_CONVERGED, STALLED, Fp64Problem, _cuda,  # noqa: F401
                            _handle, _labels, _pack, _seg_sum, _sphere_max_diag, _stats, _torch, ext, f32)
from test_newton_prox import WEIGHT_SCALES, _phi, _weights, weight_ok
from test_pcg_device import (CHUNK, CONVERGED, MAXITER, NEGCURV, NEGCURV_FIRST, ZERO_RHS, _shuffled_mesh, _spd,
                             batched_pcg_reference, jacobi_inverse_blocks)
from tssplat_b200.mesh import make_pack, perturb

BOUNDARY, NEGCURV_BOUNDARY = 5, 6
TR_OPTS = dict(max_iter=20, rtol=1e-2, rel_floor=1e-6, gtol=0.0, radius_init=1.0, radius_min=1e-12, radius_max=1e12,
               accept=1e-4, eta=0.9)
# steps the fp64 trust-region reference needs on its small mixed pack until every sphere it must converge is CONVERGED
# (test_tr_reference_mixed_pack): plain, AMIPS off and on, and proximal at test_newton_prox's two weight scales.  The
# GPU runs on the mixed 64 x 4096 pack may take GPU_SLACK more.  With AMIPS off the rough sphere does not converge: its
# model is good (rho ~ 1), but every full step that follows an accepted one would invert a tet the accepted step brought
# to J ~ 0+, so the rule rejects it and cuts the radius to eta alpha^ |d|_M (about 1/20), while an accepted step only
# doubles it; the radius collapses geometrically.  AMIPS, which grows without bound as J -> 0+, keeps tets off J = 0 and
# the rough sphere converges.  Those spheres must converge: every sphere with AMIPS on, the quiet ones otherwise.
TR_REF_STEPS = {"plain": 3, "amips": 13, "small": 3, "large": 2}
TR_MUST_ALL = {"amips"}


# ---------------------------------------------------------------------------------------------------------------------
# the solve and the rule in numpy


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


def new_tr_state(S):
    return [dict(radius=None, status=ACTIVE) for _ in range(S)]


def init_radius(st, bPb, o):
    """Delta_c = clamp(radius_init sqrt(b^T P b), radius_min, radius_max) on a sphere's first step; the fp32 radii."""
    for s, q in zip(st, bPb):
        if s["radius"] is None:
            s["radius"] = min(f32(o["radius_max"]), max(f32(o["radius_min"]), f32(o["radius_init"]) * float(np.sqrt(q))))
    return np.array([s["radius"] for s in st], np.float32)


def decide_tr(s, g, bd, dHd, dMd, pcg_status, dphi, ahat, o, w=0.0):
    """newton_decide_tr(_prox)_kernel in fp64; s = dict(radius, status), updated.  bd, dHd: the solve's records (fp32),
    dMd = |d|_M^2, dphi = Phi(x + d) - Phi(x), ahat the inversion-free step.  Returns (alpha, rho, pred, delta)."""
    if s["status"] != ACTIVE:
        return 0.0, 0.0, 0.0, 0.0
    if not weight_ok(w):
        s["status"] = STALLED
        return 0.0, 0.0, 0.0, 0.0
    if g <= f32(o["gtol"]):
        s["status"] = N_CONVERGED
        return 0.0, 0.0, 0.0, 0.0
    pred = bd - 0.5 * dHd
    rho = -dphi / pred if pred > 0.0 else 0.0
    dn = float(np.sqrt(dMd))
    lim = f32(o["eta"]) * float(ahat)
    flips = not (1.0 < lim)
    if flips:
        s["radius"] = min(0.25 * s["radius"], lim * dn)
    elif not rho >= 0.25:
        s["radius"] = 0.25 * dn
    elif rho > 0.75 and pcg_status in (BOUNDARY, NEGCURV_BOUNDARY):
        s["radius"] = min(2.0 * s["radius"], f32(o["radius_max"]))
    if not flips and pred > 0.0 and rho > f32(o["accept"]):
        return 1.0, rho, pred, dphi
    if s["radius"] < f32(o["radius_min"]):
        s["status"] = STALLED
    return 0.0, rho, pred, 0.0


def _problems(rng, S, m, indefinite):
    """S dense symmetric problems of size 3m with SPD 3x3 block-diagonal preconditioners (inverse diagonal blocks of
    |H|, so P^-1 is a fair scaling of H)."""
    H, P, b = [], [], []
    for c in range(S):
        A = _spd(rng, 3 * m, 0.2, 30.0)
        if indefinite:
            Q = np.linalg.qr(rng.normal(size=(3 * m, 3 * m)))[0]
            A = A - (Q[:, :3] * rng.uniform(5.0, 40.0, size=3)) @ Q[:, :3].T
        lam, V = np.linalg.eigh(A)
        absA = (V * np.abs(lam)) @ V.T
        B = np.zeros_like(A)
        for i in range(m):
            sl = slice(3 * i, 3 * i + 3)
            B[sl, sl] = np.linalg.inv(absA[sl, sl])
        H.append(A)
        P.append(B)
        b.append(rng.normal(size=3 * m))
    return H, P, b


@pytest.mark.parametrize("indefinite", [False, True], ids=["spd", "indefinite"])
def test_steihaug_reference_recurrences_and_cauchy_decrease(indefinite):
    rng = np.random.default_rng(11 + indefinite)
    S, m = 24, 10
    H, P, b = _problems(rng, S, m, indefinite)
    # radii from tiny to past the unconstrained solution's length
    dfull = batched_steihaug(H, b, P, [np.inf] * S, 200, 1e-12)
    full = np.array([np.sqrt(r["d"] @ np.linalg.solve(Pc, r["d"])) for r, Pc in zip(dfull, P)])
    radius = full * np.geomspace(1e-3, 3.0, S)
    out = batched_steihaug(H, b, P, radius, 200, 1e-12, history=True)
    seen = set()
    for c, r in enumerate(out):
        M = np.linalg.inv(P[c])
        norms = []
        for d, dMd in r["hist"]:
            direct = float(d @ M @ d)
            assert abs(dMd - direct) <= 1e-10 * max(direct, radius[c] ** 2 * 1e-6), (c, dMd, direct)
            norms.append(np.sqrt(direct))
        assert all(b2 >= a2 * (1 - 1e-12) for a2, b2 in zip(norms, norms[1:])), (c, norms)      # Steihaug: monotone
        dn = np.sqrt(float(r["d"] @ M @ r["d"]))
        assert dn <= radius[c] * (1 + 1e-12)
        if r["status"] in (BOUNDARY, NEGCURV_BOUNDARY):
            assert abs(dn - radius[c]) <= 1e-12 * radius[c], (c, dn, radius[c])
        # at least the Cauchy decrease in the scaled variables y = P^-1/2 d: 1/2 |g~| min(Delta, |g~| / |H~|)
        L = np.linalg.cholesky(P[c])
        g = np.sqrt(b[c] @ P[c] @ b[c])
        Hn = np.abs(np.linalg.eigvalsh(L.T @ H[c] @ L)).max()
        pred = b[c] @ r["d"] - 0.5 * r["d"] @ H[c] @ r["d"]
        assert pred >= 0.5 * g * min(radius[c], g / Hn) * (1 - 1e-10), (c, pred)
        seen.add(r["status"])
    assert BOUNDARY in seen and (NEGCURV_BOUNDARY in seen) == indefinite and (CONVERGED in seen) != indefinite
    # radius +inf: the plain reference exactly, negative curvature included
    ref = batched_pcg_reference(H, b, P, 200, 1e-12)
    for p, q in zip(dfull, ref):
        assert np.array_equal(p["d"], q["d"]) and p["status"] == q["status"] and p["n_hvp"] == q["n_hvp"]
    if indefinite:
        assert {q["status"] for q in ref} & {NEGCURV, NEGCURV_FIRST}
    # radius 0 (and NaN, read as 0): d = 0 on the boundary
    z = batched_steihaug(H[:2], b[:2], P[:2], [0.0, np.nan], 5, 1e-12)
    assert all(not r["d"].any() and r["status"] in (BOUNDARY, NEGCURV_BOUNDARY) for r in z)


_B = dict(g=1.0, bd=1.0, dHd=1.0, dMd=0.64, pcg_status=BOUNDARY, dphi=-0.45, ahat=np.inf)


def _rule(s, **kw):
    a = dict(_B, o=dict(TR_OPTS))
    a.update(kw)
    return decide_tr(s, **a)


def test_tr_rule_known_answers():
    # accept and expand: pred = 1 - 1/2 = 0.5, rho = 0.9 on the boundary: Delta doubles
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s) == (1.0, 0.9, 0.5, -0.45) and s == dict(radius=2.0, status=ACTIVE)
    s = dict(radius=float(np.float32(7e11)), status=ACTIVE)                  # ... up to radius_max
    _rule(s)
    assert s["radius"] == f32(1e12)
    # accept, interior (the solve converged inside): Delta unchanged
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, pcg_status=CONVERGED)[0] == 1.0 and s["radius"] == 1.0
    # rho in [1/4, 3/4]: accepted, Delta unchanged
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, dphi=-0.25)[:2] == (1.0, 0.5) and s["radius"] == 1.0
    # rho = 0.1 < 1/4: accepted (rho > accept) and Delta = |d|_M / 4 = 0.2
    s = dict(radius=1.0, status=ACTIVE)
    a, rho, _, delta = _rule(s, dphi=-0.05)
    assert a == 1.0 and abs(rho - 0.1) < 1e-15 and abs(s["radius"] - 0.2) < 1e-15 and delta == -0.05
    # rho < accept (energy up): rejected, shrunk
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, dphi=0.1)[0] == 0.0 and abs(s["radius"] - 0.2) < 1e-15 and s["status"] == ACTIVE
    # pred <= 0 (the model predicts no decrease): rho = 0, rejected, shrunk; a NaN change likewise
    for kw in (dict(dHd=3.0), dict(dphi=float("nan"))):
        s = dict(radius=1.0, status=ACTIVE)
        assert _rule(s, **kw)[0] == 0.0 and abs(s["radius"] - 0.2) < 1e-15, kw
    # the full step would invert a tet (1 >= eta alpha^): rejected whatever rho, Delta = min(Delta/4, eta alpha^ |d|_M)
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, ahat=np.float32(1.05))[0] == 0.0                         # 0.9 * 1.05 < 1
    assert abs(s["radius"] - 0.25) < 1e-15
    s = dict(radius=1.0, status=ACTIVE)
    _rule(s, ahat=np.float32(0.2))
    assert abs(s["radius"] - f32(0.9) * float(np.float32(0.2)) * 0.8) < 1e-15
    # rejected with Delta < radius_min: STALLED, and it stays frozen
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, dphi=0.1, o=dict(TR_OPTS, radius_min=0.3)) == (0.0, -0.2, 0.5, 0.0) and s["status"] == STALLED
    assert _rule(s) == (0.0, 0.0, 0.0, 0.0) and s == dict(radius=0.2, status=STALLED)
    # ... but an accepted step below radius_min keeps going
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, dphi=-0.05, o=dict(TR_OPTS, radius_min=0.3))[0] == 1.0 and s["status"] == ACTIVE
    # CONVERGED; an unusable weight STALLS
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, g=f32(1e-3), o=dict(TR_OPTS, gtol=1e-3)) == (0.0, 0.0, 0.0, 0.0) and s == dict(radius=1.0, status=N_CONVERGED)
    for w in (float("nan"), float("inf"), -1.0):
        s = dict(radius=1.0, status=ACTIVE)
        assert _rule(s, w=w) == (0.0, 0.0, 0.0, 0.0) and s == dict(radius=1.0, status=STALLED)
    # the initial radius
    st = new_tr_state(3)
    r = init_radius(st, [4.0, 0.0, 1e30], dict(TR_OPTS, radius_init=0.5, radius_min=1e-3, radius_max=1e6))
    assert r.tolist() == [1.0, f32(1e-3), f32(1e6)]


# ---------------------------------------------------------------------------------------------------------------------
# fp64 trust-region reference


def tr_reference(P, x0, n_steps, o, y=None, w=None):
    """tsb_newton_tr_step's algorithm in fp64: -grad (and the proximal pull), the diagonal blocks with the kernel's
    preconditioner on D + w I, the radius init, the Steihaug-Toint state machine on H + w I, the energy change at alpha = 1
    from the oracle's energies, its inversion cubic, the rule, the step."""
    x = np.asarray(x0, np.float64).reshape(-1).copy()
    prox = y is not None
    y = np.asarray(y, np.float64).reshape(-1) if prox else None
    w = np.asarray(w, np.float64) if prox else np.zeros(P.S)
    st = new_tr_state(P.S)
    sl = [slice(3 * P.vo[s], 3 * P.vo[s + 1]) for s in range(P.S)]
    hist = []
    for _ in range(n_steps):
        b = -P.grad(x)
        for s in range(P.S):
            if st[s]["status"] != ACTIVE or not weight_ok(w[s]):
                b[sl[s]] = 0.0
            elif prox:
                b[sl[s]] -= w[s] * (x[sl[s]] - y[sl[s]])
        H = P.hess_blocks(x)
        Pc = []
        for Hc, wc in zip(H, w):
            D = np.stack([Hc[3 * i:3 * i + 3, 3 * i:3 * i + 3] for i in range(len(Hc) // 3)])
            inv = jacobi_inverse_blocks(D + float(wc) * np.eye(3), o["rel_floor"])
            B = np.zeros((len(Hc), len(Hc)))
            for i, q in enumerate(inv):
                B[3 * i:3 * i + 3, 3 * i:3 * i + 3] = [[q[0], q[5], q[4]], [q[5], q[1], q[3]], [q[4], q[3], q[2]]]
            Pc.append(B)
        bs = [b[sl[s]] for s in range(P.S)]
        rad = init_radius(st, [float(q @ Pq @ q) for q, Pq in zip(bs, Pc)], o)
        sol = batched_steihaug([Hc + float(wc) * np.eye(len(Hc)) for Hc, wc in zip(H, w)], bs, Pc, rad, o["max_iter"], o["rtol"])
        d = np.concatenate([r["d"] for r in sol])
        E0, inv0 = P.sphere_energy(x)
        dE = P.sphere_energy(x + d)[0] - E0
        ahat = P.inversion_bound(x, d)
        step = []
        for s, r in enumerate(sol):
            ds = r["d"]
            dphi = dE[s] + (w[s] * (float(ds @ (x[sl[s]] - y[sl[s]])) + 0.5 * float(ds @ ds)) if prox and w[s] > 0 else 0.0)
            out = decide_tr(st[s], float(np.linalg.norm(bs[s])), r["b_dot_d"], r["d_H_d"], r["dMd"], r["status"], dphi, ahat[s], o,
                            w[s])
            phi0 = E0[s] + (0.5 * w[s] * float((x[sl[s]] - y[sl[s]]) @ (x[sl[s]] - y[sl[s]])) if prox else 0.0)
            step.append(dict(zip(("alpha", "rho", "pred", "delta"), out), status=st[s]["status"], radius=st[s]["radius"],
                             pcg=r["status"], inv0=inv0[s], phi0=phi0))
        for s in range(P.S):
            x[sl[s]] += step[s]["alpha"] * sol[s]["d"]
        hist.append(step)
    return x, hist


_TREF = {}


def _tr_ref(kind):
    """The small mixed pack of test_newton_lm's reference (sphere 0 at 0.35 h, with inverted tets): "plain" and
    "amips" minimise E, "small" and "large" the proximal objective anchored at the start with test_newton_prox's weights."""
    if kind not in _TREF:
        pk = make_pack(3, 256, seed=4)
        x = perturb(pk, sigma_rel=0.02, seed=1).astype(np.float64)
        rough = perturb(pk, sigma_rel=0.35, seed=3)
        x[pk.vert_offsets[0]:pk.vert_offsets[1]] = rough[pk.vert_offsets[0]:pk.vert_offsets[1]]
        x = x.astype(np.float32).astype(np.float64)
        P = Fp64Problem(pk, *COEF, C3 if kind == "amips" else 0.0)
        g0 = [np.linalg.norm(P.grad(x)[3 * P.vo[s]:3 * P.vo[s + 1]]) for s in range(P.S)]
        o = dict(TR_OPTS, gtol=1e-3 * min(g0))
        n = TR_REF_STEPS[kind] + 3
        if kind in WEIGHT_SCALES:
            H = P.hess_blocks(x.reshape(-1))
            w = np.array([np.float32(WEIGHT_SCALES[kind] * np.diag(Hc).max()) for Hc in H], np.float64)
            _TREF[kind] = (P, x, w, o, tr_reference(P, x, n, o, y=x, w=w))
        else:
            _TREF[kind] = (P, x, None, o, tr_reference(P, x, n, o))
    return _TREF[kind]


@pytest.mark.parametrize("kind", ["plain", "amips", "small", "large"])
def test_tr_reference_mixed_pack(kind):
    from scipy.optimize import minimize
    from test_hvp import hvp
    P, x0, w, o, (x, hist) = _tr_ref(kind)
    prox = w is not None
    y = x0.reshape(-1)
    wv = np.repeat(w, np.diff(P.vo) * 3) if prox else 0.0
    assert hist[0][0]["inv0"] > 0 and all(h["inv0"] == 0 for h in hist[0][1:])     # sphere 0 starts with inverted tets
    for t, step in enumerate(hist):              # the objective never increases; its change is the record's
        nxt = hist[t + 1] if t + 1 < len(hist) else None
        after_all = _phi(P, x, y, w) if prox else P.sphere_energy(x)[0]
        for s, r in enumerate(step):
            after = nxt[s]["phi0"] if nxt else after_all[s]
            assert after <= r["phi0"] + 1e-12 * abs(r["phi0"]), (t, s)
            assert abs((after - r["phi0"]) - r["delta"]) <= 1e-9 * abs(r["phi0"]), (t, s)
            if nxt:
                assert nxt[s]["inv0"] <= r["inv0"]
    pcg = {r["pcg"] for step in hist for r in step}
    conv = [next((t for t, step in enumerate(hist) if step[s]["status"] == N_CONVERGED), None) for s in range(P.S)]
    print(f"{kind}: converged at steps {conv}, solve statuses {sorted(pcg)}, "
          f"alpha {[[h['alpha'] for h in step] for step in hist]}, radius {[h['radius'] for h in hist[-1]]}")
    must = range(P.S) if kind in TR_MUST_ALL else range(1, P.S)
    assert all(conv[s] is not None and conv[s] <= TR_REF_STEPS[kind] for s in must), conv
    assert BOUNDARY in pcg or NEGCURV_BOUNDARY in pcg                      # the radius was active somewhere

    def jac(z):
        return P.grad(z) + wv * (z - y)

    gx = jac(x)
    for s in must:                                                          # stationary to gtol
        assert np.linalg.norm(gx[3 * P.vo[s]:3 * P.vo[s + 1]]) <= o["gtol"] * (1 + 1e-6), s
    if not prox:
        return

    # the fixed point against scipy's trust-region Newton-CG on Phi, with test_newton_prox's bound
    def fun(z):
        return float(_phi(P, z, y, w).sum())

    def hessp(z, p):
        return hvp(P.orc, z, p, P.c1, P.c2, P.order).reshape(-1) + wv * p

    ref = minimize(fun, y.copy(), jac=jac, hessp=hessp, method="trust-ncg", options=dict(gtol=1e-3 * o["gtol"], maxiter=500))
    gr = jac(ref.x)
    for s in must:
        sl = slice(3 * P.vo[s], 3 * P.vo[s + 1])
        gs, grs = np.linalg.norm(gx[sl]), np.linalg.norm(gr[sl])
        assert np.linalg.norm(x[sl] - ref.x[sl]) <= (gs + grs) / w[s], s


# ---------------------------------------------------------------------------------------------------------------------
# GPU


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


def _raw_solve_tr(torch, capi, ws, x, b, terms, opt, shift, radius, S):
    d = torch.empty_like(b)
    rec = torch.zeros((S, 8), dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    rc = capi.lib.tsb_pcg_solve_tr(ws._s, x.data_ptr(), b.data_ptr(), C.byref(terms), C.byref(opt),
                                   shift.data_ptr() if shift is not None else None, radius.data_ptr(), d.data_ptr(),
                                   rec.data_ptr(), None, st)
    assert rc == 0, ws._error(ws._s)
    return d, rec


@pytest.mark.gpu
@pytest.mark.parametrize("mesh", ["big", "a_veg", "shuffled"])
def test_infinite_radius_is_solve_ex(ext, mesh):
    """radius = +inf: d and the records of tsb_pcg_solve_ex bitwise, with and without a shift."""
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DevicePCG
    from _helpers import GOLDEN
    if mesh == "big":
        pk, x_np = _pack("mixed")
        V, T, kw = pk.verts, pk.tets, {}
    elif mesh == "a_veg":
        dz = np.load(GOLDEN + "/a_veg_mesh.npz")
        V, T = dz["verts"].astype(np.float32), dz["tets"].astype(np.int32)
        h = np.linalg.norm(V[T[:, 1]] - V[T[:, 0]], axis=1).mean()
        x_np, kw = (V + np.random.default_rng(6).normal(scale=0.05 * h, size=V.shape)).astype(np.float32), dict(force_global=True)
    else:
        V, T, x_np = _shuffled_mesh()
        kw = {}
    sp = _handle(ext, V, T, enable_amips=True, deterministic=True, **kw)
    sid_np, orph_np, S = _labels(V, T)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    x = _cuda(x_np)
    c1, c2 = 2e-4 / 64, 2e-4                   # small c1 with AMIPS on: quiet spheres reach negative curvature
    _, g = sp.energy_grad(x, c1, c2, 2, c3=C3)
    b = (-g).contiguous()
    planes = sp.hess_diag(x, c1, c2, 2, c3=C3)
    mu = (1e-2 * _sphere_max_diag(torch, planes, sid, orph, S)).contiguous()
    ws = DevicePCG(sp)
    inf = torch.full((S,), float("inf"), device="cuda")
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=C3)
    statuses = set()
    for shift in (None, mu):
        ws.set_blocks(planes, shift=shift)
        for check_every in (0, 7):
            a = ws.solve(x, b, c1, c2, 2, c3=C3, max_iter=60, rtol=1e-3, check_every=check_every, shift=shift)
            opt = _capi.tsb_pcg_options_t(max_iter=60, rtol=1e-3, check_every=check_every)
            d, rec = _raw_solve_tr(torch, _capi, ws, x, b, terms, opt, shift, inf, S)
            ra = torch.stack([a.rel_residual.view(torch.int32), a.b_dot_d.view(torch.int32), a.d_H_d.view(torch.int32), a.n_hvp,
                              a.status], 1)
            assert torch.equal(a.d, d) and torch.equal(ra, rec[:, :5]), (shift is None, check_every)
            r2 = ws.solve(x, b, c1, c2, 2, c3=C3, max_iter=60, rtol=1e-3, check_every=check_every, shift=shift, radius=float("inf"))
            assert torch.equal(r2.d, a.d) and torch.equal(r2.status, a.status)
            statuses |= set(a.status.cpu().tolist())
    print(f"{mesh}: statuses {sorted(statuses)}")
    assert not d[orph].any()


@pytest.mark.gpu
def test_finite_radius_norm_and_negative_curvature(ext):
    """On the mixed 64 x 4096 pack with AMIPS on and a small c1 (where the exact solve stops at negative curvature):
    |d|_M <= Delta (1 + 1e-4), on the boundary to 1e-4; with Delta = 2 |d_trunc|_M every sphere that ended at NEGCURV
    (or NEGCURV_FIRST) ends at NEGCURV_BOUNDARY and its model decrease is at least the truncated iterate's.
    The blocks use rel_floor = 1e-3: |d|_M computed from the fp32 d sees the fp32 rounding of z = P r amplified by up to
    the square of the blocks' condition number (1e6 at the default floor of 1e-6, which puts it near 1e-4); the
    recurrences, which the solve stops on, do not."""
    torch = _torch()
    from tssplat_b200.newton import DevicePCG
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    S = pk.num_spheres
    sid_np, orph_np, _ = _labels(pk.verts, pk.tets)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    x = _cuda(x_np)
    c1, c2 = 2e-4 / 64, 2e-4
    _, g = sp.energy_grad(x, c1, c2, 2, c3=C3)
    b = (-g).contiguous()
    planes = sp.hess_diag(x, c1, c2, 2, c3=C3)
    ws = DevicePCG(sp)
    inv = ws.set_blocks(planes, rel_floor=1e-3, want_inverse=True)
    kw = dict(c3=C3, max_iter=300, rtol=1e-3, check_every=25)
    ex = ws.solve(x, b, c1, c2, 2, **kw)
    neg = torch.isin(ex.status, torch.tensor([NEGCURV, NEGCURV_FIRST], device="cuda"))
    assert int(neg.sum()) >= 8, ex.status
    n_ex = _m_norm(torch, ex.d, inv, sid, orph, S)

    def model(res):
        Hd = sp.hvp(x, res.d, c1, c2, 2, c3=C3)[0]
        return _seg_sum(torch, (res.d.double() * (b.double() - 0.5 * Hd.double())).sum(1)[~orph], sid[~orph], S)

    for frac in (0.05, 0.3, 2.0):
        rad = (frac * n_ex).float().clamp(min=1e-30).contiguous()
        tr = ws.solve(x, b, c1, c2, 2, radius=rad, **kw)
        n = _m_norm(torch, tr.d, inv, sid, orph, S)
        R = rad.double()
        assert (n <= R * (1 + 1e-4)).all(), float((n / R).max())
        on = (tr.status == BOUNDARY) | (tr.status == NEGCURV_BOUNDARY)
        assert ((n[on] - R[on]).abs() <= 1e-4 * R[on]).all(), float(((n - R).abs() / R)[on].max())
        assert not torch.isin(tr.status, torch.tensor([NEGCURV, NEGCURV_FIRST], device="cuda")).any()
        print(f"radius {frac} |d_exact|_M: statuses {torch.bincount(tr.status, minlength=7).tolist()}")
        if frac == 2.0:
            assert (tr.status[neg] == NEGCURV_BOUNDARY).all(), tr.status
            m_tr, m_ex = model(tr), model(ex)
            assert (m_tr[neg] >= m_ex[neg] - 1e-6 * m_ex[neg].abs()).all()
            assert (tr.status[~neg] == ex.status[~neg]).all() and torch.equal(tr.d[~neg[sid] & ~orph], ex.d[~neg[sid] & ~orph])
        if frac == 0.05:
            assert on.all()
    # radius 0 (and NaN): d = 0
    z = ws.solve(x, b, c1, c2, 2, radius=torch.tensor([0.0, float("nan")] * (S // 2), device="cuda"), **kw)
    assert not z.d.any() and torch.isin(z.status, torch.tensor([BOUNDARY, NEGCURV_BOUNDARY], device="cuda")).all()


def _compose_tr(torch, sp, ws, x, st, c1, c2, c3, o, sid, orph, S, y=None, w=None, radius_after=None):
    """One tsb_newton_tr_step from the public calls and the numpy rule; st is updated.  After the first step the radius a
    sphere enters the solve with is the step's own record of the previous step (radius_after): the rule's |d|_M comes
    from d and the blocks, the kernel's from its recurrences, and the two differ in the last bits.  (The first step's
    radius is radius_max for every sphere: see the caller.)  Returns the new x and per sphere (alpha, rho, pred, delta,
    dMd)."""
    _, b = sp.energy_grad(x, c1, c2, 2, -1.0, c3=c3)
    keep = ~orph
    wn = w.cpu().numpy() if w is not None else np.zeros(S)
    ok = torch.tensor([s["status"] == ACTIVE and weight_ok(v) for s, v in zip(st, wn)], device="cuda")
    b = torch.where(~ok[sid][:, None] & keep[:, None], torch.zeros_like(b), b)
    if y is not None:
        pull = ok[sid] & keep & (w[sid] != 0)
        b = torch.where(pull[:, None], b + (-w)[sid][:, None] * (x - y), b)
    planes = sp.hess_diag(x, c1, c2, 2, c3=c3)
    inv = ws.set_blocks(planes, rel_floor=o["rel_floor"], shift=w, want_inverse=True)
    bd_ = b.double()
    bPb = _seg_sum(torch, (bd_ * _p_apply(inv, bd_)).sum(1)[keep], sid[keep], S).cpu().numpy()
    if radius_after is not None:
        for s, r in zip(st, radius_after):
            s["radius"] = float(r)
    rad = torch.from_numpy(init_radius(st, bPb, o)).cuda()
    res = ws.solve(x, b, c1, c2, 2, c3=c3, max_iter=o["max_iter"], rtol=o["rtol"], shift=w, radius=rad)
    ls = sp.line_search(x, res.d, [1.0], c1, c2, 2, c3=c3, per_sphere=True)
    gn = _seg_sum(torch, (b.double() ** 2).sum(1)[keep], sid[keep], S).sqrt().cpu().numpy()
    dMd = (_m_norm(torch, res.d, inv, sid, orph, S) ** 2).cpu().numpy()
    dd = _seg_sum(torch, (res.d.double() ** 2).sum(1)[keep], sid[keep], S).cpu().numpy()
    dx = _seg_sum(torch, (res.d.double() * (x.double() - y.double())).sum(1)[keep], sid[keep], S).cpu().numpy() if y is not None else dd * 0
    bd, dHd, sd, ss, ps = (t.cpu().numpy() for t in (res.b_dot_d, res.d_H_d, ls.sphere_delta[:, 0, 0], ls.sphere_max_step, res.status))
    out = []
    for c in range(S):
        wc = float(wn[c]) if weight_ok(wn[c]) else 0.0
        dphi = float(sd[c]) + (wc * (dx[c] + 0.5 * dd[c]) if wc > 0 else 0.0)
        out.append(decide_tr(st[c], float(gn[c]), float(bd[c]), float(dHd[c]), float(dMd[c]), int(ps[c]), dphi, ss[c], o, wn[c])
                   + (float(dMd[c]),))
    a = torch.tensor([r[0] for r in out], dtype=torch.float32, device="cuda")
    return ws.axpy(x, a, res.d), out


@pytest.mark.gpu
@pytest.mark.parametrize("prox", [False, True], ids=["plain", "prox"])
def test_tr_step_equals_its_composition(ext, prox):
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    sid_np, orph_np, S = _labels(pk.verts, pk.tets)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    c3 = C3
    o = dict(TR_OPTS, gtol=0.05)
    x1 = _cuda(x_np)
    y = w = None
    if prox:
        y = _cuda(perturb(pk, sigma_rel=0.01, seed=5))
        w = _weights(torch, sp.hess_diag(x1, c1, c2, 2, c3=c3), sid, orph, S, [1e-3, 1e-1, 1.0])
    # the initial radius clamped to radius_max on every sphere, so that it does not depend on how b^T P b is summed
    # (the kernel forms P b in fp32); well below every sphere's radius_init |b|_P, so the radius binds at the start
    _, g = sp.energy_grad(x1, c1, c2, 2, c3=c3)
    inv = nw.pcg.set_blocks(sp.hess_diag(x1, c1, c2, 2, c3=c3), want_inverse=True)
    gd = g.double()
    bPb = _seg_sum(torch, (gd * _p_apply(inv, gd)).sum(1)[~orph], sid[~orph], S).sqrt()
    o["radius_max"] = 0.1 * float(bPb.min())
    x2 = x1.clone()
    st = new_tr_state(S)
    seen, acc, rej = set(), 0, 0
    prev = None
    for t in range(8):
        r = nw.tr_step(x1, c1, c2, 2, c3=c3, anchor=y, weight=w, **o)
        x2, out = _compose_tr(torch, sp, nw.pcg, x2, st, c1, c2, c3, o, sid, orph, S, y=y, w=w, radius_after=prev)
        assert torch.equal(x1, x2), t
        assert r.alpha.cpu().tolist() == [q[0] for q in out], t
        assert r.status.cpu().tolist() == [s["status"] for s in st], t
        assert np.allclose(r.radius.cpu().numpy(), [s["radius"] for s in st], rtol=1e-5, atol=0), t
        assert np.allclose(r.d_norm.cpu().numpy() ** 2, [q[4] for q in out], rtol=1e-4, atol=0), t
        assert np.allclose(r.pred.cpu().numpy(), [q[2] for q in out], rtol=1e-6, atol=0), t
        prev = r.radius.cpu().numpy()
        seen |= set(r.status.cpu().tolist()) | {100 + v for v in r.pcg_status.cpu().tolist()}
        acc += int((r.alpha == 1).sum())
        rej += int(((r.alpha == 0) & (r.status == ACTIVE)).sum())
    print(f"prox={prox}: states seen {sorted(seen)}, accepted {acc}, rejected {rej}")
    assert N_CONVERGED in seen and acc > 0


def _records(torch, recs):
    return torch.cat([torch.cat([f.reshape(-1).contiguous().view(torch.int32) for f in r]) for r in recs])


@pytest.mark.gpu
def test_tr_determinism_graphs_and_independence(ext):
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    S = pk.num_spheres
    sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    o = dict(max_iter=10)
    x0 = _cuda(x_np)
    y0 = _cuda(perturb(pk, sigma_rel=0.02, seed=7))
    w0 = _weights(torch, sp.hess_diag(x0, c1, c2, 2, c3=C3), sid, torch.zeros_like(sid, dtype=torch.bool), S, [1e-3, 1e-2, 1e-1])
    N = 5

    def run(x_start, y=None, w=None):
        nw.reset()
        x = x_start.clone()
        out = _records(torch, [nw.tr_step(x, c1, c2, 2, c3=C3, anchor=y, weight=w, **o) for _ in range(N)])
        torch.cuda.synchronize()
        return x, out

    for y, w in ((None, None), (y0, w0)):
        xa, ra = run(x0, y, w)
        xb, rb = run(x0, y, w)
        assert torch.equal(xa, xb) and torch.equal(ra, rb)
        other = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(other):
            xc, rc = run(x0, y, w)
        assert torch.equal(xa, xc) and torch.equal(ra, rc)
    # 5 proximal steps captured in one graph (after the first call, which allocates), replayed with new anchor data
    yb, wb, xg = y0.clone(), w0.clone(), x0.clone()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        nw.tr_step(x0.clone(), c1, c2, 2, c3=C3, anchor=yb, weight=wb, **o)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        nw.reset()
        rg = _records(torch, [nw.tr_step(xg, c1, c2, 2, c3=C3, anchor=yb, weight=wb, **o) for _ in range(N)])
    xa, ra = run(x0, y0, w0)
    y1 = _cuda(perturb(pk, sigma_rel=0.03, seed=8))
    x1, r1 = run(x0, y1, w0)
    assert not torch.equal(x1, xa)
    for yv, xe, re in ((y0, xa, ra), (y1, x1, r1), (y0, xa, ra)):
        yb.copy_(yv)
        xg.copy_(x0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(xg, xe) and torch.equal(rg, re)
    # another start, anchor or weight for sphere 5 only: every other sphere's trajectory bitwise unchanged
    vo = pk.vert_offsets
    keep = torch.ones(len(x0), dtype=torch.bool, device="cuda")
    keep[vo[5]:vo[6]] = False
    others = torch.arange(S, device="cuda") != 5
    xs0 = x0.clone()
    xs0[vo[5]:vo[6]] += 0.01 * torch.randn_like(xs0[vo[5]:vo[6]])
    y2, w2 = y0.clone(), w0.clone()
    y2[vo[5]:vo[6]] += 0.01 * torch.randn_like(y2[vo[5]:vo[6]])
    w2[5] *= 3.0
    for xv, yv, wv, yr in ((xs0, None, None, None), (x0, y2, w0, y0), (x0, y0, w2, y0)):
        nw.reset()
        xs = xv.clone()
        recs = [nw.tr_step(xs, c1, c2, 2, c3=C3, anchor=yv, weight=wv, **o) for _ in range(N)]
        nw.reset()
        xr = x0.clone()
        refs = [nw.tr_step(xr, c1, c2, 2, c3=C3, anchor=yr, weight=w0 if yr is not None else None, **o) for _ in range(N)]
        assert torch.equal(xs[keep], xr[keep]) and not torch.equal(xs[~keep], xr[~keep])
        for p, q in zip(recs, refs):
            for f in p._fields:
                assert torch.equal(getattr(p, f)[others], getattr(q, f)[others]), f


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(warps_per_cta=8), dict(warps_per_cta=16), dict(force_global=True), dict(psd=True)],
                         ids=["w8", "w16", "global", "psd"])
def test_tr_handle_variants_and_orphans(ext, kw):
    """Orphan vertices never move; E falls on every sphere; with proximal weights, a NaN (sphere 0) and a negative one
    (sphere 1) freeze just that sphere as STALLED.  "psd": one step over a projected-Hessian workspace."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    V, T, x_np = _shuffled_mesh()
    kw = dict(kw)
    psd = kw.pop("psd", False)
    sp = _handle(ext, V, T, deterministic=True, **kw)
    sid_np, orph_np, S = _labels(V, T)
    assert S == 3
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    c1, c2 = COEF
    nw = DeviceNewton(sp, hessian="psd" if psd else None)
    x = _cuda(x_np)
    x0 = x.clone()
    e0 = sp.energy_grad_spheres(x0, c1, c2, 2, want_grad=False)[2]
    for t in range(1 if psd else 4):
        r = nw.tr_step(x, c1, c2, 2)
        assert torch.equal(x[orph], x0[orph]) and (r.delta <= 0).all() and not torch.isnan(x).any()
    assert (r.alpha == 1).all() or t > 0
    e1 = sp.energy_grad_spheres(x, c1, c2, 2, want_grad=False)[2]
    assert ((c1 * e1.smooth + c2 * e1.barrier) < (c1 * e0.smooth + c2 * e0.barrier)).all()
    if psd:
        assert not torch.isin(r.pcg_status, torch.tensor([NEGCURV, NEGCURV_FIRST], device="cuda")).any()
        return
    nw.reset()
    x = x0.clone()
    y = (x0 + 0.01 * torch.randn_like(x0)).contiguous()
    w = torch.tensor([float("nan"), -1e-3, 1e-3], device="cuda")
    for t in range(4):
        r = nw.tr_step(x, c1, c2, 2, anchor=y, weight=w)
        assert torch.equal(x[orph], x0[orph])
        assert r.status[:2].tolist() == [STALLED, STALLED] and r.alpha[:2].tolist() == [0.0, 0.0]
    frozen = (sid < 2) & ~orph
    assert torch.equal(x[frozen], x0[frozen]) and not torch.equal(x[sid == 2], x0[sid == 2])


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_tr_convergence_mixed_pack(ext, amips):
    """The mixed 64 x 4096 pack through SmoothnessBarrierEnergy.newton_step with FLAGS.newton_method = "tr": every
    step's change is <= 0 and a fresh sphere_stats launch agrees with the start plus the summed deltas (AMIPS on: on the
    quiet spheres, as in test_newton_lm); the quiet spheres gain no inverted tet and each ends CONVERGED (|g_c| down by
    1e3) within the fp64 reference's step count plus GPU_SLACK; the rough spheres gain at most MAX_ROUNDING_FLIPS tets
    per step and lose inverted tets overall."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("mixed")
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000,
                                                        amips_coeff=C3 if amips else 0.0, deterministic=True, newton_method="tr"))
    x = torch.nn.Parameter(_cuda(x_np))
    it = 0
    e_start, inv_start = _stats(E, x, it)
    g0 = E.newton_step(x.detach().clone(), it, max_iter=1).grad_norm
    E.device_newton.reset()
    quiet = torch.arange(pk.num_spheres, device="cuda") % 4 != 0
    gtol = 1e-3 * float(g0[quiet].min())
    acc = torch.zeros(pk.num_spheres, dtype=torch.float64, device="cuda")
    inv_prev = inv_start
    n = TR_REF_STEPS["amips" if amips else "plain"] + GPU_SLACK
    done = None
    for t in range(n):
        r = E.newton_step(x, it, gtol=gtol)
        assert (r.delta <= 0).all(), t
        acc += r.delta.double()
        e, inv = _stats(E, x, it)
        tol = 1e-4 * e_start.abs()
        err = (e - e_start - acc).abs()
        checked = quiet if amips else torch.ones_like(quiet)
        assert (err[checked] <= tol[checked]).all(), (t, float((err / tol)[checked].max()))
        assert (inv[quiet] <= inv_prev[quiet]).all(), t
        assert int((inv - inv_prev).clamp(min=0).max()) <= MAX_ROUNDING_FLIPS, t
        inv_prev = inv
        if done is None and bool((r.status[quiet] == N_CONVERGED).all()):
            done = t + 1
    assert int(inv[~quiet].sum()) < int(inv_start[~quiet].sum())
    print(f"amips={amips}: quiet spheres converged after {done} steps (allowed {n}); status {r.status.cpu().tolist()}; "
          f"radius {float(r.radius.min()):.3e}..{float(r.radius.max()):.3e}")
    assert (r.status[quiet] == N_CONVERGED).all(), r.status


@pytest.mark.gpu
def test_tr_bookkeeping_and_argument_errors(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DeviceNewton, DevicePCG
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    ws = DevicePCG(sp)
    nw = DeviceNewton(sp, ws)
    n, S = sp.n, nw.n_spheres
    rows = int(np.diff(pk.vert_offsets).sum())
    chunks = int(sum(-(-int(m) // CHUNK) for m in np.diff(pk.vert_offsets)))
    pcg0 = 72 * n + 4 * rows + 36 * chunks + 64 * S + 4 * (S + 1) + 4
    nw0 = 48 * n + 24 * chunks + 172 * S + 176
    assert ws.device_bytes == pcg0 and nw.device_bytes == nw0
    c1, c2 = COEF
    x = _cuda(x_np)
    y = x.clone()
    w = torch.full((S,), 1e-3, device="cuda")
    E = _capi.TSB_E_INVALID
    st = torch.cuda.current_stream().cuda_stream
    L = _capi.lib
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=0.0)
    # the first trust-region step allocates: refused inside a capture (which survives), then made outside it
    graph = torch.cuda.CUDAGraph()
    g = x.clone()
    with torch.cuda.graph(graph):
        g.add_(1.0)
        with pytest.raises(RuntimeError, match="capture"):
            nw.tr_step(g, c1, c2, 2)
        with pytest.raises(RuntimeError, match="capture"):
            ws.solve(g, g, c1, c2, 2, radius=1.0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g, x + 1.0)
    assert int(L.tsb_pcg_device_bytes(ws._s)) == pcg0 and nw.device_bytes == nw0
    z = x.clone()
    for bad in (dict(max_iter=0), dict(rtol=-1.0), dict(rel_floor=float("nan")), dict(gtol=-1.0), dict(radius_init=0.0),
                dict(radius_init=float("inf")), dict(radius_min=0.0), dict(radius_min=2.0, radius_max=1.0),
                dict(radius_max=float("inf")), dict(accept=0.25), dict(accept=-1.0), dict(accept=float("nan")), dict(eta=0.0),
                dict(eta=1.5)):
        o = nw.tr_options(**bad)
        assert L.tsb_newton_tr_step(nw._nw, z.data_ptr(), None, None, C.byref(terms), C.byref(o), None, st) == E, bad
    o = nw.tr_options()
    o.reserved[6] = 1
    assert L.tsb_newton_tr_step(nw._nw, z.data_ptr(), None, None, C.byref(terms), C.byref(o), None, st) == E
    o = nw.tr_options()
    for args in ((None, z.data_ptr(), None, None, C.byref(terms), C.byref(o)),
                 (nw._nw, None, None, None, C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), y.data_ptr(), None, C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), None, w.data_ptr(), C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), z.data_ptr(), w.data_ptr(), C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), None, None, None, C.byref(o)),
                 (nw._nw, z.data_ptr(), None, None, C.byref(terms), None),
                 (nw._nw, z.data_ptr(), None, None, C.byref(_capi.tsb_terms_t(c1=c1, c2=c2, order=3)), C.byref(o))):
        assert L.tsb_newton_tr_step(*args, None, st) == E
    popt = _capi.tsb_pcg_options_t(max_iter=5, rtol=1e-3, check_every=0)
    d = torch.empty_like(x)
    assert L.tsb_pcg_solve_tr(ws._s, x.data_ptr(), x.data_ptr(), C.byref(terms), C.byref(popt), None, None, d.data_ptr(), None,
                              None, st) == E
    with pytest.raises(TypeError):
        nw.tr_options(tau=1.0)
    with pytest.raises(ValueError):
        nw.minimize(z, 1, c1, c2, 2, method="cg")
    torch.cuda.synchronize()
    assert torch.equal(z, x)
    assert int(L.tsb_pcg_device_bytes(ws._s)) == pcg0 and nw.device_bytes == nw0
    # after the first (plain) step: 32 bytes per sphere on the solver workspace, 20 on the Newton workspace; a proximal
    # one adds the d.(x - y) partials
    r = nw.tr_step(z, c1, c2, 2)
    assert int(L.tsb_pcg_device_bytes(ws._s)) == pcg0 + 32 * S and nw.device_bytes == nw0 + 20 * S
    nw.tr_step(z.clone(), c1, c2, 2, anchor=y, weight=w)
    assert nw.device_bytes == nw0 + 20 * S + 8 * chunks
    # reset re-arms the radius: the same first step again
    nw.reset()
    z2 = x.clone()
    r2 = nw.tr_step(z2, c1, c2, 2)
    assert torch.equal(z, z2) and torch.equal(r.radius, r2.radius) and torch.equal(r.rho, r2.rho)
    assert (r.radius > 0).all() and (r.d_norm > 0).all()


@pytest.mark.gpu
def test_module_tr_route(ext):
    """FLAGS.newton_method = "tr" routes newton_step and prox_step to the trust-region step; absent, they stay LM."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    from tssplat_b200.newton import DeviceNewton, NewtonStepResult, NewtonTRStepResult
    pk, x_np = _pack("small")
    flags = dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000, deterministic=True)
    it = 5
    E_lm = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    E_tr = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(flags, newton_method="tr"))
    xa, xb = torch.nn.Parameter(_cuda(x_np)), torch.nn.Parameter(_cuda(x_np))
    assert isinstance(E_lm.newton_step(xa, it), NewtonStepResult)
    assert isinstance(E_tr.newton_step(xb, it), NewtonTRStepResult)
    y = _cuda(perturb(pk, sigma_rel=0.01, seed=5))
    r = E_tr.prox_step(xb, y, it, 1e-2, n_steps=3, max_iter=15)
    assert isinstance(r, NewtonTRStepResult) and (r.alpha > 0).any()
    # the same three proximal steps through DeviceNewton.minimize on a second handle
    E2 = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    nw = DeviceNewton(E2.tet_sp)
    c1, c2 = E2.coeff_scheduler(it)
    z = _cuda(x_np)
    nw.tr_step(z, c1, c2, E2.order_at(it))
    nw.reset()
    n, r2 = nw.minimize(z, 3, c1, c2, E2.order_at(it), anchor=y, weight=1e-2, method="tr", max_iter=15)
    assert n == 3 and torch.equal(z, xb.detach()) and torch.equal(r2.radius, r.radius)
    with pytest.raises(ValueError, match="newton_method"):
        SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(flags, newton_method="cg")).newton_step(xa, it)
