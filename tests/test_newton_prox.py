"""The proximal Newton step: tsb_newton_prox_step, DeviceNewton.step/minimize(anchor=, weight=) and
SmoothnessBarrierEnergy.prox_step, which minimise Phi_c(x) = E_c(x) + (w_c / 2) |x_c - y_c|^2 per sphere.

CPU: the step's decision rule with the proximal terms as a numpy function with known answers; an fp64 proximal LM
reference (dense per-sphere H + w I from the matrix-form HVPs, the oracle's energies and inversion cubic) on a small
mixed pack, whose fixed point is checked against scipy's trust-region Newton-CG on Phi and which pins the step counts
the GPU runs are allowed.  GPU: w = 0 is tsb_newton_step bitwise; one step against the public calls composed with the
numpy rule; convergence and the anchor bound on the mixed 64 x 4096 pack against the fp64 oracle; determinism, graph
replays with new anchors and weights, independence; handle variants, orphans, invalid weights, argument errors; the
module route."""
import ctypes as C

import numpy as np
import pytest

# ext: test_newton_lm's module-scoped fixture, requested by name
from test_newton_lm import (ACTIVE, ALPHAS, C3, COEF, GPU_SLACK, N_CONVERGED, OPTS, STALLED, Fp64Problem, _cuda,  # noqa: F401
                            _handle, _labels, _pack, _seg_sum, _sphere_max_diag, _torch, decide, ext, f32, new_state)
from test_pcg_device import CHUNK, _shuffled_mesh, batched_pcg_reference, jacobi_inverse_blocks
from tssplat_b200.mesh import make_pack, perturb

# steps the fp64 proximal reference needs on its small mixed pack until every sphere it must converge is CONVERGED, per
# weight scale (test_prox_reference_mixed_pack); the GPU runs may take GPU_SLACK more.  Under the large weight the rough
# sphere is held near an anchor with inverted tets: its minimiser keeps tets at J ~ 0, where the order-2 barrier's
# curvature jumps, and the step sizes keep cycling without meeting gtol (Phi still falls at every step)
PROX_REF_STEPS = {"small": 12, "large": 2}
WEIGHT_SCALES = {"small": 1e-4, "large": 10.0}     # times the sphere's largest Hessian diagonal entry at the start


# ---------------------------------------------------------------------------------------------------------------------
# the proximal rule in numpy


def weight_ok(w):
    return bool(np.isfinite(w) and w >= 0)


def init_mu_prox(st, maxD, w, o):
    """mu_c = tau (max (D_v)_ii + w_c) on a sphere's first step, clamped; returns the fp32 shifts mu_c + w_c (w_c read as
    0 where it is unusable)."""
    out = []
    for s, m, wc in zip(st, maxD, w):
        we = float(np.float32(wc)) if weight_ok(wc) else 0.0
        if s["mu"] is None:
            s["mu"] = min(f32(o["mu_max"]), max(f32(o["mu_min"]), f32(o["tau"]) * (float(m) + we)))
            s["nu"] = 2.0
        out.append(s["mu"] + we)
    return np.array(out, np.float32)


def decide_prox(s, g, bd, dHd, mu_f, dd, dE, ahat, o, w, dx, alphas=ALPHAS):
    """decide of test_newton_lm with the proximal terms (newton_decide_kernel<true> in fp64): dPhi_k = dE_k + w (a_k dx +
    a_k^2 dd / 2) in place of dE_k, pred with mu' = mu_f - w; an unusable w freezes the sphere as STALLED.  dx = d.(x - y).
    Returns (alpha, k, dPhi of the step, rho)."""
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


_BASE = dict(g=1.0, bd=1.0, dHd=1.5, mu_f=1.0, dd=1.0, dE=[-0.5] + [-0.3 * 2.0 ** -k for k in range(1, 8)], ahat=np.inf)


def _prule(s, w=0.0, dx=0.0, **kw):
    a = dict(_BASE, o=dict(OPTS))
    a.update(kw)
    return decide_prox(s, w=w, dx=dx, **a)


def test_prox_rule_known_answers():
    # w = 0 is the plain rule, on every branch decide's known answers exercise
    cases = [dict(dE=[-0.75] + [-0.1] * 7), dict(dE=[-1.5] + [-0.1] * 7), dict(dE=[0.2, -0.2] + [-0.01] * 6),
             dict(ahat=np.float32(0.3)), dict(dE=[1.0] * 8), dict(bd=-1.0, dE=[-5.0] * 8), dict(bd=1.0, dHd=10.0, dd=0.0),
             dict(g=f32(1e-3), o=dict(OPTS, gtol=1e-3))]
    for kw in cases:
        s1, s2 = dict(mu=3.0, nu=2.0, status=ACTIVE), dict(mu=3.0, nu=2.0, status=ACTIVE)
        a = dict(_BASE, o=dict(OPTS))
        a.update(kw)
        assert _prule(s1, w=0.0, dx=0.7, **kw) == decide(s2, **a) and s1 == s2, kw
    # the quadratic term turns a rejected step into an accepted one: dE = +0.1 everywhere, but w (d.(x-y) + dd/2) =
    # 1 * (-1 + 0.5) gives dPhi_0 = -0.4; pred = 1 - (1.5 - (1 - 1) * 1) / 2 = 0.25, rho = 0.4 / 0.25 = 1.6
    s = dict(mu=3.0, nu=8.0, status=ACTIVE)
    assert _prule(dict(mu=3.0, nu=8.0, status=ACTIVE), dE=[0.1] * 8)[:2] == (0.0, -1)
    a, k, d, rho = _prule(s, w=1.0, dx=-1.0, dE=[0.1] * 8)
    assert (a, k) == (1.0, 0) and abs(d + 0.4) < 1e-15 and abs(rho - 1.6) < 1e-15
    assert s == dict(mu=1.0, nu=2.0, status=ACTIVE)                                # rho > 1: mu / 3
    # ... and back: an accepted full step (dE_0 = -0.5) rejected once the step leaves the anchor (dx = 0.5, w = 2):
    # dPhi_k = dE_k + 2 (a/2 + a^2/2) > 0 down to a = 1/8, and at a = 1/16 dPhi = -0.1 + 2 (1/32 + 1/512) < 0
    dE = [-0.5, -0.3, -0.2] + [-0.1] * 5
    assert _prule(dict(mu=1.0, nu=2.0, status=ACTIVE), dE=dE)[:2] == (1.0, 0)
    s = dict(mu=1.0, nu=2.0, status=ACTIVE)
    a, k, d, rho = _prule(s, w=2.0, dx=0.5, mu_f=3.0, dE=dE)
    assert (a, k) == (1.0 / 16, 4) and abs(d - (-0.1 + 2.0 * (0.5 / 16 + 0.5 / 256))) < 1e-15
    # pred uses mu' = mu_f - w = 1: 1 - (1.5 - 1) / 2 = 0.75; dPhi_0 = -0.5 + 2 = 1.5, rho = -2; mu * nu
    assert abs(rho + 2.0) < 1e-15 and s == dict(mu=2.0, nu=4.0, status=ACTIVE)
    # pred with mu': shift 3 = mu + w with w = 2 models H + 2 I; dPhi_0 = -1.75 + 2 * 0.5 = -0.75 = -pred: rho = 1
    s = dict(mu=3.0, nu=2.0, status=ACTIVE)
    assert _prule(s, w=2.0, dx=0.0, mu_f=3.0, dE=[-1.75] + [-0.1] * 7) == (1.0, 0, -0.75, 1.0) and s["mu"] == 1.0
    # the shift itself: mu = tau (max D + w), shift = fp32(mu + w)
    st = new_state(2)
    sh = init_mu_prox(st, [np.float32(4.0), np.float32(1.0)], [np.float32(0.5), np.float32(np.nan)], OPTS)
    assert st[0]["mu"] == f32(1e-3) * 4.5 and sh[0] == np.float32(st[0]["mu"] + 0.5)
    assert st[1]["mu"] == f32(1e-3) * 1.0 and sh[1] == np.float32(st[1]["mu"])
    # an unusable weight: no step, STALLED, mu untouched, and it stays frozen
    for w in (float("nan"), float("inf"), -1e-3):
        s = dict(mu=1.0, nu=2.0, status=ACTIVE)
        assert _prule(s, w=w, dE=[-0.75] + [-0.1] * 7) == (0.0, -1, 0.0, 0.0)
        assert s == dict(mu=1.0, nu=2.0, status=STALLED)
        assert _prule(s, w=1.0, dE=[-0.75] + [-0.1] * 7) == (0.0, -1, 0.0, 0.0) and s["status"] == STALLED


# ---------------------------------------------------------------------------------------------------------------------
# fp64 proximal LM reference


def prox_lm_reference(P, x0, y, w, n_steps, o):
    """tsb_newton_prox_step's algorithm in fp64 (lm_reference of test_newton_lm with the proximal terms)."""
    x = np.asarray(x0, np.float64).reshape(-1).copy()
    y = np.asarray(y, np.float64).reshape(-1)
    st = new_state(P.S)
    sl = [slice(3 * P.vo[s], 3 * P.vo[s + 1]) for s in range(P.S)]
    hist = []
    for _ in range(n_steps):
        b = -P.grad(x)
        for s in range(P.S):
            if st[s]["status"] != ACTIVE or not weight_ok(w[s]):
                b[sl[s]] = 0.0
            else:
                b[sl[s]] -= w[s] * (x[sl[s]] - y[sl[s]])
        H = P.hess_blocks(x)
        D = [np.stack([Hc[3 * i:3 * i + 3, 3 * i:3 * i + 3] for i in range(len(Hc) // 3)]) for Hc in H]
        shift = init_mu_prox(st, [Dc[:, [0, 1, 2], [0, 1, 2]].max() for Dc in D], w, o)
        Pc = []
        for Dc, m in zip(D, shift):
            inv = jacobi_inverse_blocks(Dc + float(m) * np.eye(3), o["rel_floor"])
            B = np.zeros((3 * len(Dc), 3 * len(Dc)))
            for i, q in enumerate(inv):
                B[3 * i:3 * i + 3, 3 * i:3 * i + 3] = [[q[0], q[5], q[4]], [q[5], q[1], q[3]], [q[4], q[3], q[2]]]
            Pc.append(B)
        bs = [b[sl[s]] for s in range(P.S)]
        sol = batched_pcg_reference([Hc + float(m) * np.eye(len(Hc)) for Hc, m in zip(H, shift)], bs, Pc, o["max_iter"], o["rtol"])
        d = np.concatenate([r["d"] for r in sol])
        E0, inv0 = P.sphere_energy(x)
        dE = np.stack([P.sphere_energy(x + a * d)[0] - E0 for a in ALPHAS[:o["n_alpha"]]], axis=1)
        ahat = P.inversion_bound(x, d)
        step = []
        for s, r in enumerate(sol):
            ds = sol[s]["d"]
            out = decide_prox(st[s], float(np.linalg.norm(bs[s])), r["b_dot_d"], r["d_H_d"], shift[s], float(ds @ ds), dE[s],
                              ahat[s], o, w[s], float(ds @ (x[sl[s]] - y[sl[s]])))
            step.append(dict(zip(("alpha", "k", "delta", "rho"), out), status=st[s]["status"], inv0=inv0[s],
                             phi0=E0[s] + 0.5 * w[s] * float((x[sl[s]] - y[sl[s]]) @ (x[sl[s]] - y[sl[s]]))))
        for s in range(P.S):
            x[sl[s]] += step[s]["alpha"] * sol[s]["d"]
        hist.append(step)
    return x, hist


_PREF = {}


def _prox_ref(scale):
    """The small mixed pack of test_newton_lm's reference (sphere 0 at 0.35 h, with inverted tets), AMIPS off, started
    at x = y, with w_c = scale times the sphere's largest Hessian diagonal entry at the start."""
    if scale not in _PREF:
        pk = make_pack(3, 256, seed=4)
        x = perturb(pk, sigma_rel=0.02, seed=1).astype(np.float64)
        rough = perturb(pk, sigma_rel=0.35, seed=3)
        x[pk.vert_offsets[0]:pk.vert_offsets[1]] = rough[pk.vert_offsets[0]:pk.vert_offsets[1]]
        x = x.astype(np.float32).astype(np.float64)
        P = Fp64Problem(pk, *COEF, 0.0)
        H = P.hess_blocks(x.reshape(-1))
        w = np.array([np.float32(WEIGHT_SCALES[scale] * np.diag(Hc).max()) for Hc in H], np.float64)
        g0 = [np.linalg.norm(P.grad(x)[3 * P.vo[s]:3 * P.vo[s + 1]]) for s in range(P.S)]
        o = dict(OPTS, gtol=1e-3 * min(g0))
        _PREF[scale] = (P, x, w, o, prox_lm_reference(P, x, x, w, PROX_REF_STEPS["small"] + 3, o))
    return _PREF[scale]


def _phi(P, x, y, w):
    E, _ = P.sphere_energy(x)
    r = (np.asarray(x, np.float64) - y).reshape(-1, 3)
    return E + 0.5 * w * np.array([(r[P.vo[s]:P.vo[s + 1]] ** 2).sum() for s in range(P.S)])


@pytest.mark.parametrize("scale", ["small", "large"])
def test_prox_reference_mixed_pack(scale):
    from scipy.optimize import minimize
    from test_hvp import hvp
    P, y, w, o, (x, hist) = _prox_ref(scale)
    wv = np.repeat(w, np.diff(P.vo) * 3)
    for t, step in enumerate(hist):                                  # Phi never increases; its change is the record's
        phi1 = hist[t + 1] if t + 1 < len(hist) else None
        for s, r in enumerate(step):
            after = phi1[s]["phi0"] if phi1 else _phi(P, x, y.reshape(-1), w)[s]
            assert after <= r["phi0"] + 1e-12 * abs(r["phi0"]), (t, s)
            assert abs((after - r["phi0"]) - r["delta"]) <= 1e-9 * abs(r["phi0"]), (t, s)
    conv = [next((t for t, step in enumerate(hist) if step[s]["status"] == N_CONVERGED), None) for s in range(P.S)]
    print(f"{scale}: converged at steps {conv}, w {w}, k {[[h['k'] for h in step] for step in hist]}")
    must = range(P.S) if scale == "small" else range(1, P.S)
    assert all(conv[s] is not None and conv[s] <= PROX_REF_STEPS[scale] for s in must), conv
    # the fixed point against an independent minimiser of Phi: scipy's trust-region Newton-CG with the oracle's fp64
    # gradient and the matrix-form HVP, from the same start
    yf = y.reshape(-1)

    def fun(z):
        return float(_phi(P, z, yf, w).sum())

    def jac(z):
        return P.grad(z) + wv * (z - yf)

    def hessp(z, p):
        return hvp(P.orc, z, p, P.c1, P.c2, P.order).reshape(-1) + wv * p

    ref = minimize(fun, yf.copy(), jac=jac, hessp=hessp, method="trust-ncg", options=dict(gtol=1e-3 * o["gtol"], maxiter=500))
    # both points are stationary to gtol, and Phi_c is w_c-strongly convex where H_c is PSD, so per sphere
    # |x_c - x*_c| <= (|grad Phi_c(x)| + |grad Phi_c(x*)|) / w_c; Phi_c agrees to that distance times the gradients
    gx, gr = jac(x), jac(ref.x)
    for s in must:
        sl = slice(3 * P.vo[s], 3 * P.vo[s + 1])
        gs, grs = np.linalg.norm(gx[sl]), np.linalg.norm(gr[sl])
        assert gs <= o["gtol"] * (1 + 1e-6), (s, gs, o["gtol"])
        dist = np.linalg.norm(x[sl] - ref.x[sl])
        print(f"sphere {s}: |x - x*| = {dist:.3e}, bound {(gs + grs) / w[s]:.3e}, |x* - y| = {np.linalg.norm(ref.x[sl] - yf[sl]):.3e}")
        assert dist <= (gs + grs) / w[s], s
        phis, phir = _phi(P, x, yf, w)[s], _phi(P, ref.x, yf, w)[s]
        assert abs(phis - phir) <= (gs + grs) * (gs + grs) / w[s] + 1e-12 * abs(phir), (s, phis, phir)
    if scale == "large":                         # the dominant weight holds x near the anchor; the small one does not
        sp, (xs, _) = _prox_ref("small")[0], _prox_ref("small")[4]
        assert np.abs(x - yf).max() < 0.2 * np.abs(xs - yf).max()


# ---------------------------------------------------------------------------------------------------------------------
# GPU


def _weights(torch, planes, sid, orph, S, scales):
    """w_c = scales[c % len(scales)] times the sphere's largest diagonal entry, float32 [S]."""
    mx = _sphere_max_diag(torch, planes, sid, orph, S)
    sc = torch.tensor(scales, dtype=torch.float32, device="cuda").repeat(S // len(scales) + 1)[:S]
    return (mx * sc).contiguous()


def _records(torch, recs):
    return torch.cat([torch.cat([f.reshape(-1).contiguous().view(torch.int32) for f in r]) for r in recs])


@pytest.mark.gpu
@pytest.mark.parametrize("c3", [0.0, C3], ids=["amips-off", "amips-on"])
def test_zero_weight_is_newton_step(ext, c3):
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    x1, x2 = _cuda(x_np), _cuda(x_np)
    y = _cuda(perturb(pk, sigma_rel=0.1, seed=9))           # far from x: w = 0 must ignore it
    w = torch.zeros(nw.n_spheres, device="cuda")
    a = [nw.step(x1, c1, c2, 2, c3=c3, max_iter=10) for _ in range(6)]
    nw.reset()
    b = [nw.step(x2, c1, c2, 2, c3=c3, anchor=y, weight=w, max_iter=10) for _ in range(6)]
    assert torch.equal(x1, x2)
    assert torch.equal(_records(torch, a), _records(torch, b))
    assert (a[-1].alpha > 0).any()


def _compose_prox(torch, sp, ws, x, y, w, st, c1, c2, c3, o, sid, orph, S):
    """One tsb_newton_prox_step from the public calls and the numpy rule; st is updated.  Returns the new x and per
    sphere (alpha, k, dPhi, rho)."""
    _, b = sp.energy_grad(x, c1, c2, 2, -1.0, c3=c3)
    wn = w.cpu().numpy()
    ok = torch.tensor([s["status"] == ACTIVE and weight_ok(v) for s, v in zip(st, wn)], device="cuda")
    keep = ~orph
    b = torch.where(~ok[sid][:, None] & keep[:, None], torch.zeros_like(b), b)
    pull = ok[sid] & keep & (w[sid] != 0)
    b = torch.where(pull[:, None], b + (-w)[sid][:, None] * (x - y), b)
    planes = sp.hess_diag(x, c1, c2, 2, c3=c3)
    shift = torch.from_numpy(init_mu_prox(st, _sphere_max_diag(torch, planes, sid, orph, S).cpu().numpy(), wn, o)).cuda()
    ws.set_blocks(planes, rel_floor=o["rel_floor"], shift=shift)
    res = ws.solve(x, b, c1, c2, 2, c3=c3, max_iter=o["max_iter"], rtol=o["rtol"], shift=shift)
    ls = sp.line_search(x, res.d, ALPHAS[:o["n_alpha"]], c1, c2, 2, c3=c3, per_sphere=True)
    gn = _seg_sum(torch, (b.double() ** 2).sum(1)[keep], sid[keep], S).sqrt().cpu().numpy()
    dd = _seg_sum(torch, (res.d.double() ** 2).sum(1)[keep], sid[keep], S).cpu().numpy()
    dx = _seg_sum(torch, (res.d.double() * (x.double() - y.double())).sum(1)[keep], sid[keep], S).cpu().numpy()
    bd, dHd, sd, ss = (t.cpu().numpy() for t in (res.b_dot_d, res.d_H_d, ls.sphere_delta[:, :, 0], ls.sphere_max_step))
    out = [decide_prox(st[c], float(gn[c]), float(bd[c]), float(dHd[c]), shift[c].item(), float(dd[c]), sd[c], ss[c], o,
                       wn[c], float(dx[c])) for c in range(S)]
    a = torch.tensor([r[0] for r in out], dtype=torch.float32, device="cuda")
    return ws.axpy(x, a, res.d), out


@pytest.mark.gpu
@pytest.mark.parametrize("c3", [0.0, C3], ids=["amips-off", "amips-on"])
def test_prox_step_equals_its_composition(ext, c3):
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    sid_np, orph_np, S = _labels(pk.verts, pk.tets)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    x1 = _cuda(x_np)
    y = _cuda(perturb(pk, sigma_rel=0.01, seed=5))          # an anchor a little off the start
    w = _weights(torch, sp.hess_diag(x1, c1, c2, 2, c3=c3), sid, orph, S, [1e-3, 1e-1, 1.0])
    o = dict(OPTS, gtol=0.05)
    x2 = x1.clone()
    st = new_state(S)
    seen = set()
    for t in range(6):
        r = nw.step(x1, c1, c2, 2, c3=c3, anchor=y, weight=w, **o)
        x2, out = _compose_prox(torch, sp, nw.pcg, x2, y, w, st, c1, c2, c3, o, sid, orph, S)
        assert torch.equal(x1, x2), t
        assert r.k.cpu().tolist() == [q[1] for q in out] and r.alpha.cpu().tolist() == [q[0] for q in out], t
        assert r.status.cpu().tolist() == [s["status"] for s in st], t
        assert np.allclose(r.mu.cpu().numpy(), [s["mu"] for s in st], rtol=1e-12, atol=0)
        took = np.array([q[1] >= 0 for q in out])
        assert np.allclose(r.delta.cpu().numpy()[took], [q[2] for q in out if q[1] >= 0], rtol=1e-5, atol=0)
        seen |= set(r.status.cpu().tolist())
    assert N_CONVERGED in seen


def _oracle_phi(P, x, y, w, grad=False):
    """fp64 per-sphere E_c and |x_c - y_c|^2 / 2 from the oracle; grad: also |grad Phi_c| and |grad E_c|."""
    x = x.double().cpu().numpy().reshape(-1)
    E, _ = P.sphere_energy(x)
    r = x - y
    sl = [slice(3 * P.vo[s], 3 * P.vo[s + 1]) for s in range(P.S)]
    q = np.array([0.5 * float(r[s_] @ r[s_]) for s_ in sl])
    if not grad:
        return E, q
    gE = P.grad(x)
    g = gE + np.repeat(w, np.diff(P.vo) * 3) * r
    return E, q, np.array([np.linalg.norm(g[s_]) for s_ in sl]), np.array([np.linalg.norm(gE[s_]) for s_ in sl])


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_prox_convergence_mixed_pack(ext, amips):
    """The mixed 64 x 4096 pack through SmoothnessBarrierEnergy.prox_step, started at x = y, weights that differ between
    spheres (1e-4 .. 1 times the sphere's largest Hessian diagonal entry): every step's dPhi <= 0; the fp64 oracle's Phi_c
    agrees with the start plus the summed deltas (tolerance as in test_newton_lm.test_convergence_mixed_pack, with AMIPS
    on the quiet spheres only); every quiet sphere ends CONVERGED; at the end the oracle's |grad E_c + w_c (x_c - y_c)|
    is at most gtol plus the parity gate's 1e-5 |grad E_c|."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("mixed")
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000,
                                                        amips_coeff=C3 if amips else 0.0, deterministic=True))
    it = 0
    c1, c2 = E.coeff_scheduler(it)
    x = torch.nn.Parameter(_cuda(x_np))
    y = x.detach().clone()
    S = pk.num_spheres
    sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
    w = _weights(torch, E.hess_diag(x, it), sid, torch.zeros_like(sid, dtype=torch.bool), S, [1e-4, 1e-3, 1e-2, 1e-1, 1.0])
    P = Fp64Problem(pk, c1, c2, E.amips_coeff)
    yn = y.double().cpu().numpy().reshape(-1)
    wn = w.double().cpu().numpy()
    e0, q0, g0, _ = _oracle_phi(P, x.detach(), yn, wn, grad=True)
    phi_start = e0 + wn * q0
    quiet = np.arange(S) % 4 != 0
    gtol = 1e-3 * float(g0[quiet].min())
    acc = np.zeros(S)
    n = max(PROX_REF_STEPS.values()) + GPU_SLACK
    for t in range(n):
        r = E.prox_step(x, y, it, w, restart=(t == 0), gtol=gtol)
        d = r.delta.double().cpu().numpy()
        assert (d <= 0).all(), t
        acc += d
        e, q = _oracle_phi(P, x.detach(), yn, wn)
        tol = 1e-4 * np.abs(phi_start)
        err = np.abs(e + wn * q - phi_start - acc)
        checked = quiet if amips else np.ones(S, bool)
        assert (err[checked] <= tol[checked]).all(), (t, float((err / tol)[checked].max()))
    st = r.status.cpu().numpy()
    print(f"amips={amips}: status {st.tolist()}, gtol {gtol:.3e}")
    assert (st[quiet] == N_CONVERGED).all(), st
    _, _, gphi, gE = _oracle_phi(P, x.detach(), yn, wn, grad=True)
    assert (gphi[quiet] <= gtol + 1e-5 * gE[quiet]).all(), float((gphi[quiet] / (gtol + 1e-5 * gE[quiet])).max())


@pytest.mark.gpu
def test_anchor_bound(ext):
    """Started at x = y, each accepted step lowers Phi_c, so (w_c / 2) |x_c - y_c|^2 <= E_c(y) - E_c(x) at every step
    (fp64 oracle, with fp32 slack); with weights from 1e-4 to 10 times the largest diagonal entry, the heavily weighted
    quiet spheres stay an order of magnitude closer to the anchor than the others."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, deterministic=True)
    S = pk.num_spheres
    sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
    c1, c2 = COEF
    x = _cuda(x_np)
    y = x.clone()
    scales = [1e-4, 1e-2, 10.0]
    w = _weights(torch, sp.hess_diag(x, c1, c2, 2), sid, torch.zeros_like(sid, dtype=torch.bool), S, scales)
    nw = DeviceNewton(sp)
    P = Fp64Problem(pk, c1, c2, 0.0)
    yn = y.double().cpu().numpy().reshape(-1)
    wn = w.double().cpu().numpy()
    Ey, _ = P.sphere_energy(yn)
    slack = 1e-5 * np.abs(Ey)
    for t in range(10):
        nw.step(x, c1, c2, 2, anchor=y, weight=w, max_iter=10)
        xn = x.double().cpu().numpy().reshape(-1)
        Ex, _ = P.sphere_energy(xn)
        r = (xn - yn).reshape(-1, 3)
        q = np.array([(r[pk.vert_offsets[s]:pk.vert_offsets[s + 1]] ** 2).sum() for s in range(S)])
        assert (0.5 * wn * q <= Ey - Ex + slack).all(), (t, float((0.5 * wn * q - (Ey - Ex)).max()))
    disp = np.sqrt(q / np.diff(pk.vert_offsets))
    grp, quiet = np.arange(S) % len(scales), np.arange(S) % 4 != 0
    med = [np.median(disp[(grp == g) & quiet]) for g in range(len(scales))]
    print(f"rms displacement of the quiet spheres per weight scale {dict(zip(scales, med))}")
    assert med[-1] < 0.1 * min(med[:-1])


@pytest.mark.gpu
def test_prox_determinism_graphs_and_independence(ext):
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

    def run(y, w):
        nw.reset()
        x = x0.clone()
        out = _records(torch, [nw.step(x, c1, c2, 2, c3=C3, anchor=y, weight=w, **o) for _ in range(N)])
        torch.cuda.synchronize()
        return x, out

    xa, ra = run(y0, w0)
    xb, rb = run(y0.clone(), w0.clone())
    assert torch.equal(xa, xb) and torch.equal(ra, rb)
    other = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(other):
        xc, rc = run(y0, w0)
    assert torch.equal(xa, xc) and torch.equal(ra, rc)
    # N steps captured in one graph with anchor and weight buffers; replayed after new data is copied into them
    yb, wb, xg = y0.clone(), w0.clone(), x0.clone()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):                              # warm-up outside the capture (allocator)
        nw.step(x0.clone(), c1, c2, 2, c3=C3, anchor=yb, weight=wb, **o)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        nw.reset()
        rg = _records(torch, [nw.step(xg, c1, c2, 2, c3=C3, anchor=yb, weight=wb, **o) for _ in range(N)])
    y1 = _cuda(perturb(pk, sigma_rel=0.03, seed=8))
    w1 = (w0 * torch.linspace(0.5, 2.0, S, device="cuda")).contiguous()
    x1, r1 = run(y1, w1)
    assert not torch.equal(x1, xa)
    for yv, wv, xe, re in ((y0, w0, xa, ra), (y1, w1, x1, r1), (y0, w0, xa, ra)):
        yb.copy_(yv)
        wb.copy_(wv)
        xg.copy_(x0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(xg, xe) and torch.equal(rg, re)
    # another anchor and weight for sphere 5 only: every other sphere's trajectory bitwise unchanged
    vo = pk.vert_offsets
    y2, w2 = y0.clone(), w0.clone()
    y2[vo[5]:vo[6]] += 0.01 * torch.randn_like(y2[vo[5]:vo[6]])
    w2[5] *= 3.0
    for yv, wv in ((y2, w0), (y0, w2)):
        nw.reset()
        xs = x0.clone()
        recs = [nw.step(xs, c1, c2, 2, c3=C3, anchor=yv, weight=wv, **o) for _ in range(N)]
        nw.reset()
        xr = x0.clone()
        refs = [nw.step(xr, c1, c2, 2, c3=C3, anchor=y0, weight=w0, **o) for _ in range(N)]
        keep = torch.ones(len(x0), dtype=torch.bool, device="cuda")
        keep[vo[5]:vo[6]] = False
        others = torch.arange(S, device="cuda") != 5
        assert torch.equal(xs[keep], xr[keep]) and not torch.equal(xs[~keep], xr[~keep])
        for p, q in zip(recs, refs):
            for f in p._fields:
                assert torch.equal(getattr(p, f)[others], getattr(q, f)[others]), f


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(warps_per_cta=8), dict(warps_per_cta=16), dict(force_global=True)], ids=["w8", "w16", "global"])
def test_prox_handle_variants_orphans_and_invalid_weights(ext, kw):
    """Orphan vertices never move; a NaN weight (sphere 0) and a negative one (sphere 1) freeze just that sphere as
    STALLED, unmoved; the third sphere steps and its Phi falls."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    V, T, x_np = _shuffled_mesh()
    sp = _handle(ext, V, T, deterministic=True, **kw)
    assert sp.info["mode_global"] == int(bool(kw.get("force_global")))
    sid_np, orph_np, S = _labels(V, T)
    assert S == 3
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    x = _cuda(x_np)
    x0 = x.clone()
    y = (x0 + 0.01 * torch.randn_like(x0)).contiguous()
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    w = torch.tensor([float("nan"), -1e-3, 1e-3], device="cuda")
    for t in range(6):
        r = nw.step(x, c1, c2, 2, anchor=y, weight=w)
        assert torch.equal(x[orph], x0[orph])
        assert r.status[:2].tolist() == [STALLED, STALLED] and r.alpha[:2].tolist() == [0.0, 0.0]
        assert (r.delta <= 0).all() and not torch.isnan(x).any()
        assert float(r.alpha[2]) > 0 or t > 0
    frozen = (sid < 2) & ~orph
    assert torch.equal(x[frozen], x0[frozen]) and not torch.equal(x[sid == 2], x0[sid == 2])


@pytest.mark.gpu
def test_prox_argument_errors_and_bookkeeping(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    nw = DeviceNewton(sp)
    n, S = sp.n, nw.n_spheres
    chunks = int(sum(-(-int(m) // CHUNK) for m in np.diff(pk.vert_offsets)))
    assert nw.device_bytes == 48 * n + 24 * chunks + 172 * S + 176
    c1, c2 = COEF
    x = _cuda(x_np)
    y = x.clone()
    w = torch.full((S,), 1e-3, device="cuda")
    E = _capi.TSB_E_INVALID
    st = torch.cuda.current_stream().cuda_stream
    L = _capi.lib
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=0.0)
    z = x.clone()
    # the first proximal step allocates: refused inside a capture (which survives), then made outside it
    graph = torch.cuda.CUDAGraph()
    g = x.clone()
    with torch.cuda.graph(graph):
        g.add_(1.0)
        with pytest.raises(RuntimeError, match="capture"):
            nw.step(g, c1, c2, 2, anchor=y, weight=w)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g, x + 1.0)
    assert nw.device_bytes == 48 * n + 24 * chunks + 172 * S + 176
    for bad in (dict(max_iter=0), dict(rtol=-1.0), dict(tau=0.0), dict(mu_min=2.0, mu_max=1.0), dict(sigma=1.0), dict(eta=0.0),
                dict(n_alpha=9)):
        o = nw.options(**bad)
        assert L.tsb_newton_prox_step(nw._nw, z.data_ptr(), y.data_ptr(), w.data_ptr(), C.byref(terms), C.byref(o), None, st) == E, bad
    o = nw.options()
    o.reserved[0] = 1
    assert L.tsb_newton_prox_step(nw._nw, z.data_ptr(), y.data_ptr(), w.data_ptr(), C.byref(terms), C.byref(o), None, st) == E
    o = nw.options()
    for args in ((None, z.data_ptr(), y.data_ptr(), w.data_ptr(), C.byref(terms), C.byref(o)),
                 (nw._nw, None, y.data_ptr(), w.data_ptr(), C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), None, w.data_ptr(), C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), y.data_ptr(), None, C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), z.data_ptr(), w.data_ptr(), C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), y.data_ptr(), w.data_ptr(), None, C.byref(o)),
                 (nw._nw, z.data_ptr(), y.data_ptr(), w.data_ptr(), C.byref(terms), None),
                 (nw._nw, z.data_ptr(), y.data_ptr(), w.data_ptr(), C.byref(_capi.tsb_terms_t(c1=c1, c2=c2, order=3)), C.byref(o))):
        assert L.tsb_newton_prox_step(*args, None, st) == E
    torch.cuda.synchronize()
    assert torch.equal(z, x)
    # Python checks
    with pytest.raises(RuntimeError, match="not be x"):
        nw.step(z, c1, c2, 2, anchor=z, weight=w)
    with pytest.raises(RuntimeError, match="needs an anchor"):
        nw.step(z, c1, c2, 2, weight=w)
    with pytest.raises(RuntimeError, match="needs a weight"):
        nw.step(z, c1, c2, 2, anchor=y)
    with pytest.raises(RuntimeError, match="weight"):
        nw.step(z, c1, c2, 2, anchor=y, weight=torch.ones(S + 1, device="cuda"))
    with pytest.raises(RuntimeError, match="anchor"):
        nw.step(z, c1, c2, 2, anchor=y.double(), weight=w)
    torch.cuda.synchronize()
    assert torch.equal(z, x)
    # after the first proximal step the workspace holds 8 bytes per chunk more; a float weight is every sphere's
    r = nw.step(z, c1, c2, 2, anchor=y, weight=1e-3)
    assert nw.device_bytes == 48 * n + 24 * chunks + 172 * S + 176 + 8 * chunks
    nw.reset()
    z2 = x.clone()
    r2 = nw.step(z2, c1, c2, 2, anchor=y, weight=w)
    assert torch.equal(z, z2) and torch.equal(r.mu, r2.mu)


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_module_prox_step(ext, amips):
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("small")
    flags = dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000, deterministic=True,
                 amips_coeff=C3 if amips else 0.0)
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    it = 5
    c1, c2 = E.coeff_scheduler(it)
    x = torch.nn.Parameter(_cuda(x_np))
    y = _cuda(perturb(pk, sigma_rel=0.01, seed=5))
    r = E.prox_step(x, y, it, 1e-2, n_steps=3, max_iter=15)
    assert E.device_newton.pcg is E.device_pcg and (r.alpha > 0).any() and not torch.equal(x.detach(), _cuda(x_np))
    # the same three steps on a second module's handle through DeviceNewton.minimize
    E2 = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    nw = DeviceNewton(E2.tet_sp)
    z = _cuda(x_np)
    n, r2 = nw.minimize(z, 3, c1, c2, E2.order_at(it), c3=E2.amips_coeff, anchor=y, weight=1e-2, max_iter=15)
    assert n == 3 and torch.equal(z, x.detach()) and torch.equal(r2.mu, r.mu)
    # restart: with every sphere frozen (gtol huge), restart=False leaves x alone; restart=True starts them again
    E.prox_step(x, y, it, 1e-2, gtol=1e30)
    x1 = x.detach().clone()
    r = E.prox_step(x, y, it, 1e-2, restart=False)
    assert torch.equal(x.detach(), x1) and (r.status == N_CONVERGED).all()
    r = E.prox_step(x, y, it, 1e-2, n_steps=2)
    assert not torch.equal(x.detach(), x1) and (r.alpha > 0).any()
