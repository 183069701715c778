"""The backtracking trust-region Newton step: tsb_newton_tr_step_ex with a tsb_newton_backtrack_t,
DeviceNewton.trls_step / minimize(method="trls") and SmoothnessBarrierEnergy with FLAGS.newton_method = "trls".

CPU: the step's decision rule in numpy with known answers (full step, backtracked after a flip or a poor model, no
Armijo step, bd <= 0, STALLED, an unusable weight, the radius clamp); an fp64 reference on the small mixed pack, plain,
AMIPS on and proximal at two weight scales, which pins the step counts the GPU runs are allowed and whose fixed points
are checked for stationarity (and, proximal, against scipy's trust-region Newton-CG).  GPU: one step against the public
calls composed with the numpy rule; bt == NULL is tsb_newton_tr_step bitwise, and spheres that never backtrack follow
the trust-region step's trajectory bitwise; determinism, graph replays and independence; every backtracked step's
Armijo decrease and inversion bound; handle variants, orphans and the projected Hessian; convergence on the mixed
64 x 4096 pack; bookkeeping and argument errors; the module route."""
import ctypes as C

import numpy as np
import pytest

# ext: test_newton_lm's module-scoped fixture, requested by name
from test_newton_lm import (ACTIVE, C3, COEF, GPU_SLACK, MAX_ROUNDING_FLIPS, N_CONVERGED, STALLED, Fp64Problem, _cuda,  # noqa: F401
                            _handle, _labels, _pack, _seg_sum, _stats, _torch, ext, f32)
from test_newton_prox import WEIGHT_SCALES, _phi, _weights, weight_ok
from test_newton_tr import (BOUNDARY, NEGCURV_BOUNDARY, TR_OPTS, TR_REF_STEPS, _m_norm, _p_apply, _records, batched_steihaug,
                            init_radius, new_tr_state)
from test_pcg_device import CHUNK, NEGCURV, NEGCURV_FIRST, _shuffled_mesh, jacobi_inverse_blocks
from tssplat_b200.mesh import make_pack, perturb

TRLS_OPTS = dict(TR_OPTS, n_alpha=8, sigma=1e-4)
ALPHAS = [2.0 ** -k for k in range(8)]
# steps the fp64 reference needs on its small mixed pack until every sphere is CONVERGED (test_trls_reference_mixed_pack),
# as TR_REF_STEPS for the trust-region step; the GPU runs on the mixed 64 x 4096 pack may take GPU_SLACK more.  Unlike the
# trust-region step's reference, this one converges the rough sphere with AMIPS off as well.
# With the large proximal weight the rough sphere does not converge here either: the anchor holds it next to its
# inverted start, every full step would invert a tet (eta alpha^ between 0.01 and 0.96), each step is backtracked to
# 2^-k on a boundary solve, so the radius becomes max(2^-k |d|_M, Delta / 4) = 2^-k Delta and still shrinks
# geometrically (to radius_min after 29 steps, then STALLED).  The quiet spheres must converge in every variant.
TRLS_REF_STEPS = {"plain": 5, "amips": 13, "small": 10, "large": 2}
TRLS_MUST_ALL = {"plain", "amips", "small"}


# ---------------------------------------------------------------------------------------------------------------------
# the rule in numpy


def decide_trls(s, g, bd, dHd, dMd, pcg_status, dphi, ahat, o, w=0.0):
    """newton_decide_trls(_prox)_kernel in fp64; s = dict(radius, status), updated.  As test_newton_tr.decide_tr, but
    dphi[k] = Phi(x + 2^-k d) - Phi(x) for k < n_alpha: a step the trust-region rule rejects is backtracked to the largest
    2^-k (k >= 1) below eta alpha^ with the Armijo decrease, and the radius then becomes max(2^-k |d|_M, Delta / 4),
    clamped.  Returns (alpha, rho, pred, delta)."""
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
        for k in range(1, int(o["n_alpha"])):
            a = ALPHAS[k]
            if a < lim and dphi[k] <= -f32(o["sigma"]) * a * bd:
                s["radius"] = min(f32(o["radius_max"]), max(f32(o["radius_min"]), max(a * dn, 0.25 * old)))
                return a, rho, pred, dphi[k]
    s["radius"] = new
    if new < f32(o["radius_min"]):
        s["status"] = STALLED
    return 0.0, rho, pred, 0.0


# dphi(a) = -a + a^2 / 4 along d with bd = 1, dHd = 1/2 (a quadratic model that is exact): pred = 0.75, rho = 1
_DPHI = [-a + 0.25 * a * a for a in ALPHAS]
_B = dict(g=1.0, bd=1.0, dHd=0.5, dMd=0.64, pcg_status=BOUNDARY, dphi=_DPHI, ahat=np.inf)


def _rule(s, **kw):
    a = dict(_B, o=dict(TRLS_OPTS))
    a.update(kw)
    return decide_trls(s, **a)


def test_trls_rule_known_answers():
    # full step taken: rho = 1 on the boundary, Delta doubles, as the trust-region rule
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s) == (1.0, 1.0, 0.75, _DPHI[0]) and s == dict(radius=2.0, status=ACTIVE)
    # backtracked after a flip: eta alpha^ = 0.9 * 0.2 = 0.18, so 1/8 is the largest 2^-k below it (1/4 is not);
    # Delta = max(|d|_M / 8, Delta / 4) = max(0.1, 0.25), where the trust-region rule would cut it to 0.18 * 0.8 = 0.144
    s = dict(radius=1.0, status=ACTIVE)
    a, rho, pred, delta = _rule(s, ahat=np.float32(0.2))
    assert (a, rho, pred, delta) == (0.125, 1.0, 0.75, _DPHI[3]) and s == dict(radius=0.25, status=ACTIVE)
    s = dict(radius=0.2, status=ACTIVE)                                      # ... and |d|_M alpha when that is larger
    _rule(s, ahat=np.float32(0.2))
    assert s["radius"] == 0.1
    # backtracked after rho <= accept: the full step raises Phi, half of it satisfies Armijo; Delta = max(0.4, 0.25)
    dphi = [0.1, -0.3] + _DPHI[2:]
    s = dict(radius=1.0, status=ACTIVE)
    a, rho, _, delta = _rule(s, dphi=dphi)
    assert a == 0.5 and delta == -0.3 and abs(rho + 0.1 / 0.75) < 1e-15 and s == dict(radius=0.4, status=ACTIVE)
    # pred <= 0 (rho = 0): backtracking still runs on the Armijo test alone
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, dHd=3.0, dphi=dphi)[:3] == (0.5, 0.0, -0.5)
    # no Armijo step: every 2^-k raises Phi, or decreases it by less than sigma alpha bd -> the trust-region rejection
    for dp in ([0.1] * 8, [0.1] + [-f32(1e-4) * a * 0.5 for a in ALPHAS[1:]]):
        s = dict(radius=1.0, status=ACTIVE)
        assert _rule(s, dphi=dp)[0] == 0.0 and abs(s["radius"] - 0.2) < 1e-15 and s["status"] == ACTIVE
    # an Armijo step at 1/2 that is not below eta alpha^ (0.9 * 0.5 = 0.45): the next one, 1/4
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, dphi=dphi, ahat=np.float32(0.5))[0] == 0.25
    # n_alpha = 2 tries 1/2 only
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, ahat=np.float32(0.5), o=dict(TRLS_OPTS, n_alpha=2))[0] == 0.0 and abs(s["radius"] - 0.25) < 1e-15
    # bd <= 0: no backtracking, whatever the changes
    for bd in (0.0, -1.0):
        s = dict(radius=1.0, status=ACTIVE)
        assert _rule(s, bd=bd, dphi=dphi)[0] == 0.0 and abs(s["radius"] - 0.2) < 1e-15
    # STALLED below radius_min when nothing is taken; a backtracked step below it keeps going (and lifts the radius)
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, dphi=[0.1] * 8, o=dict(TRLS_OPTS, radius_min=0.3))[0] == 0.0 and s["status"] == STALLED
    assert _rule(s) == (0.0, 0.0, 0.0, 0.0) and s == dict(radius=0.2, status=STALLED)
    s = dict(radius=0.2, status=ACTIVE)
    assert _rule(s, ahat=np.float32(0.2), o=dict(TRLS_OPTS, radius_min=0.3))[0] == 0.125
    assert s == dict(radius=f32(0.3), status=ACTIVE)
    # the clamp from above: max(alpha |d|_M, Delta / 4) > radius_max
    s = dict(radius=8.0, status=ACTIVE)
    _rule(s, ahat=np.float32(0.2), o=dict(TRLS_OPTS, radius_max=1.5))
    assert s["radius"] == f32(1.5)
    # an unusable weight STALLS; CONVERGED
    for w in (float("nan"), float("inf"), -1.0):
        s = dict(radius=1.0, status=ACTIVE)
        assert _rule(s, w=w) == (0.0, 0.0, 0.0, 0.0) and s == dict(radius=1.0, status=STALLED)
    s = dict(radius=1.0, status=ACTIVE)
    assert _rule(s, g=f32(1e-3), o=dict(TRLS_OPTS, gtol=1e-3)) == (0.0, 0.0, 0.0, 0.0) and s["status"] == N_CONVERGED


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference


def trls_reference(P, x0, n_steps, o, y=None, w=None):
    """tsb_newton_tr_step_ex's algorithm in fp64: test_newton_tr.tr_reference with the energy change at every 2^-k,
    k < n_alpha, and decide_trls."""
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
        dE = np.stack([P.sphere_energy(x + a * d)[0] - E0 for a in ALPHAS[:o["n_alpha"]]], 1)
        ahat = P.inversion_bound(x, d)
        step = []
        for s, r in enumerate(sol):
            ds = r["d"]
            dphi = [dE[s, k] + (w[s] * (a * float(ds @ (x[sl[s]] - y[sl[s]])) + 0.5 * a * a * float(ds @ ds)) if prox and w[s] > 0
                                else 0.0) for k, a in enumerate(ALPHAS[:o["n_alpha"]])]
            rad_in = st[s]["radius"]
            out = decide_trls(st[s], float(np.linalg.norm(bs[s])), r["b_dot_d"], r["d_H_d"], r["dMd"], r["status"], dphi, ahat[s],
                              o, w[s])
            phi0 = E0[s] + (0.5 * w[s] * float((x[sl[s]] - y[sl[s]]) @ (x[sl[s]] - y[sl[s]])) if prox else 0.0)
            step.append(dict(zip(("alpha", "rho", "pred", "delta"), out), status=st[s]["status"], radius=st[s]["radius"],
                             radius_in=rad_in, ahat=float(ahat[s]), pcg=r["status"], inv0=inv0[s], phi0=phi0, bd=r["b_dot_d"],
                             dphi=dphi))
        for s in range(P.S):
            x[sl[s]] += step[s]["alpha"] * sol[s]["d"]
        hist.append(step)
    return x, hist


_REF = {}
REF_EXTRA = 3                 # steps past the pinned count the reference runs (the fixed point must hold)


def _trls_ref(kind, n=None):
    """test_newton_tr._tr_ref's setup (the small mixed pack, sphere 0 at 0.35 h with inverted tets) under the
    backtracking rule."""
    key = (kind, n)
    if key not in _REF:
        pk = make_pack(3, 256, seed=4)
        x = perturb(pk, sigma_rel=0.02, seed=1).astype(np.float64)
        rough = perturb(pk, sigma_rel=0.35, seed=3)
        x[pk.vert_offsets[0]:pk.vert_offsets[1]] = rough[pk.vert_offsets[0]:pk.vert_offsets[1]]
        x = x.astype(np.float32).astype(np.float64)
        P = Fp64Problem(pk, *COEF, C3 if kind == "amips" else 0.0)
        g0 = [np.linalg.norm(P.grad(x)[3 * P.vo[s]:3 * P.vo[s + 1]]) for s in range(P.S)]
        o = dict(TRLS_OPTS, gtol=1e-3 * min(g0))
        n = TRLS_REF_STEPS[kind] + REF_EXTRA if n is None else n
        if kind in WEIGHT_SCALES:
            H = P.hess_blocks(x.reshape(-1))
            w = np.array([np.float32(WEIGHT_SCALES[kind] * np.diag(Hc).max()) for Hc in H], np.float64)
            _REF[key] = (P, x, w, o, trls_reference(P, x, n, o, y=x, w=w))
        else:
            _REF[key] = (P, x, None, o, trls_reference(P, x, n, o))
    return _REF[key]


@pytest.mark.parametrize("kind", ["plain", "amips", "small", "large"])
def test_trls_reference_mixed_pack(kind):
    from scipy.optimize import minimize
    from test_hvp import hvp
    P, x0, w, o, (x, hist) = _trls_ref(kind)
    prox = w is not None
    y = x0.reshape(-1)
    wv = np.repeat(w, np.diff(P.vo) * 3) if prox else 0.0
    assert hist[0][0]["inv0"] > 0 and all(h["inv0"] == 0 for h in hist[0][1:])     # sphere 0 starts with inverted tets
    n_back = 0
    for t, step in enumerate(hist):              # the objective never increases; its change is the record's
        nxt = hist[t + 1] if t + 1 < len(hist) else None
        after_all = _phi(P, x, y, w) if prox else P.sphere_energy(x)[0]
        for s, r in enumerate(step):
            after = nxt[s]["phi0"] if nxt else after_all[s]
            assert after <= r["phi0"] + 1e-12 * abs(r["phi0"]), (t, s)
            assert abs((after - r["phi0"]) - r["delta"]) <= 1e-9 * abs(r["phi0"]), (t, s)
            if 0.0 < r["alpha"] < 1.0:           # backtracked: Armijo below the inversion bound
                n_back += 1
                assert r["alpha"] < f32(o["eta"]) * r["ahat"] and r["delta"] <= -f32(o["sigma"]) * r["alpha"] * r["bd"], (t, s)
            if nxt and s > 0:
                assert nxt[s]["inv0"] <= r["inv0"]
    conv = [next((t for t, step in enumerate(hist) if step[s]["status"] == N_CONVERGED), None) for s in range(P.S)]
    print(f"{kind}: converged at steps {conv} (trust region: {TR_REF_STEPS[kind]}), backtracked steps {n_back}, "
          f"sphere 0: alpha {[step[0]['alpha'] for step in hist]}, eta alpha^ "
          f"{[round(f32(o['eta']) * step[0]['ahat'], 3) for step in hist]}, radius {[float(f'{step[0]['radius']:.3g}') for step in hist]}")
    assert n_back > 0
    must = range(P.S) if kind in TRLS_MUST_ALL else range(1, P.S)
    assert all(conv[s] is not None and conv[s] <= TRLS_REF_STEPS[kind] for s in must), conv
    assert all(conv[s] <= TR_REF_STEPS[kind] for s in range(1, P.S)), conv     # quiet spheres: within the TR counts
    if kind == "plain":
        assert hist[-1][0]["inv0"] == 0

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


def _compose_trls(torch, sp, ws, x, st, c1, c2, c3, o, sid, orph, S, y=None, w=None, radius_after=None):
    """One tsb_newton_tr_step_ex from the public calls and decide_trls (test_newton_tr._compose_tr with the line search
    at every 2^-k); st is updated.  Returns the new x and per sphere (alpha, rho, pred, delta, dMd, ahat, bd, dphi)."""
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
    na = o["n_alpha"]
    ls = sp.line_search(x, res.d, ALPHAS[:na], c1, c2, 2, c3=c3, per_sphere=True)
    gn = _seg_sum(torch, (b.double() ** 2).sum(1)[keep], sid[keep], S).sqrt().cpu().numpy()
    dMd = (_m_norm(torch, res.d, inv, sid, orph, S) ** 2).cpu().numpy()
    dd = _seg_sum(torch, (res.d.double() ** 2).sum(1)[keep], sid[keep], S).cpu().numpy()
    dx = _seg_sum(torch, (res.d.double() * (x.double() - y.double())).sum(1)[keep], sid[keep], S).cpu().numpy() if y is not None else dd * 0
    bd, dHd, sd, ss, ps = (t.cpu().numpy() for t in (res.b_dot_d, res.d_H_d, ls.sphere_delta[:, :, 0], ls.sphere_max_step, res.status))
    out = []
    for c in range(S):
        wc = float(wn[c]) if weight_ok(wn[c]) else 0.0
        dphi = [float(sd[c, k]) + (wc * (a * dx[c] + 0.5 * a * a * dd[c]) if wc > 0 else 0.0) for k, a in enumerate(ALPHAS[:na])]
        out.append(decide_trls(st[c], float(gn[c]), float(bd[c]), float(dHd[c]), float(dMd[c]), int(ps[c]), dphi, ss[c], o, wn[c])
                   + (float(dMd[c]), float(ss[c]), float(bd[c]), dphi))
    a = torch.tensor([r[0] for r in out], dtype=torch.float32, device="cuda")
    return ws.axpy(x, a, res.d), out


@pytest.mark.gpu
@pytest.mark.parametrize("prox", [False, True], ids=["plain", "prox"])
def test_trls_step_equals_its_composition(ext, prox):
    """Eight steps on the small pack against the public calls and the numpy rule: the same alpha and status, the radius
    to 1e-5, bitwise the same x; every backtracked step satisfies the Armijo decrease below eta alpha^."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    sid_np, orph_np, S = _labels(pk.verts, pk.tets)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    c3 = C3
    o = dict(TRLS_OPTS, gtol=0.05)
    x1 = _cuda(x_np)
    y = w = None
    if prox:      # anchored at the start: the pull holds the rough sphere near its inverted tets, so it backtracks
        y = x1.clone()
        w = _weights(torch, sp.hess_diag(x1, c1, c2, 2, c3=c3), sid, orph, S, [1e-3, 1e-1, 1.0])
    # the initial radius clamped to radius_max on every sphere (as test_tr_step_equals_its_composition)
    _, g = sp.energy_grad(x1, c1, c2, 2, c3=c3)
    inv = nw.pcg.set_blocks(sp.hess_diag(x1, c1, c2, 2, c3=c3), want_inverse=True)
    gd = g.double()
    bPb = _seg_sum(torch, (gd * _p_apply(inv, gd)).sum(1)[~orph], sid[~orph], S).sqrt()
    o["radius_max"] = 0.1 * float(bPb.min())
    x2 = x1.clone()
    st = new_tr_state(S)
    seen, full, back, rej = set(), 0, 0, 0
    prev = None
    for t in range(8):
        r = nw.trls_step(x1, c1, c2, 2, c3=c3, anchor=y, weight=w, **o)
        x2, out = _compose_trls(torch, sp, nw.pcg, x2, st, c1, c2, c3, o, sid, orph, S, y=y, w=w, radius_after=prev)
        assert torch.equal(x1, x2), t
        alpha = r.alpha.cpu().tolist()
        assert alpha == [q[0] for q in out], t
        assert r.status.cpu().tolist() == [s["status"] for s in st], t
        assert np.allclose(r.radius.cpu().numpy(), [s["radius"] for s in st], rtol=1e-5, atol=0), t
        assert np.allclose(r.pred.cpu().numpy(), [q[2] for q in out], rtol=1e-6, atol=0), t
        delta = r.delta.cpu().numpy()
        for c, q in enumerate(out):
            a = q[0]
            if 0.0 < a < 1.0:
                k = ALPHAS.index(a)
                assert a < f32(o["eta"]) * q[5] and q[7][k] <= -f32(o["sigma"]) * a * q[6], (t, c)
                assert abs(delta[c] - q[7][k]) <= 1e-6 * abs(q[7][k]) + 1e-12, (t, c)
        prev = r.radius.cpu().numpy()
        seen |= set(r.status.cpu().tolist())
        full += alpha.count(1.0)
        back += sum(0.0 < a < 1.0 for a in alpha)
        rej += int(((r.alpha == 0) & (r.status == ACTIVE)).sum())
    print(f"prox={prox}: states seen {sorted(seen)}, full steps {full}, backtracked {back}, rejected {rej}")
    assert N_CONVERGED in seen and full > 0 and back > 0


def _raw_tr(torch, capi, nw, x, terms, opt, bt, S, ex=True):
    """tsb_newton_tr_step_ex (ex) or tsb_newton_tr_step on the current stream; the raw [S, 16] records."""
    rec = torch.zeros((S, 16), dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    if ex:
        rc = capi.lib.tsb_newton_tr_step_ex(nw._nw, x.data_ptr(), None, None, C.byref(terms), C.byref(opt),
                                            C.byref(bt) if bt is not None else None, rec.data_ptr(), st)
    else:
        rc = capi.lib.tsb_newton_tr_step(nw._nw, x.data_ptr(), None, None, C.byref(terms), C.byref(opt), rec.data_ptr(), st)
    assert rc == 0, nw._error(nw._nw)
    return rec


def _bits(torch, r, S):
    """[S, k] int32 view of every field of a NewtonTRStepResult."""
    return torch.cat([getattr(r, f).contiguous().view(torch.int32).reshape(S, -1) for f in r._fields], 1)


@pytest.mark.gpu
def test_trls_without_backtracking_is_tr(ext):
    """bt == NULL: tsb_newton_tr_step's x and records bitwise.  On the mixed 64 x 4096 pack, the trust-region and the
    backtracking step side by side, AMIPS off and on: every sphere whose full step was accepted at every step so far
    (or that converged) has a bitwise-identical trajectory and records, so the line search's alpha = 1 change does not
    depend on n_alpha."""
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    S = pk.num_spheres
    sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
    c1, c2 = COEF
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=0.0)
    na, nb = DeviceNewton(sp), DeviceNewton(sp)
    opt = na.tr_options(max_iter=10)
    xa, xb = _cuda(x_np), _cuda(x_np)
    for t in range(4):
        ra = _raw_tr(torch, _capi, na, xa, terms, opt, None, S, ex=False)
        rb = _raw_tr(torch, _capi, nb, xb, terms, opt, None, S)
        assert torch.equal(xa, xb) and torch.equal(ra, rb), t
    for c3 in (0.0, C3):
        ntr, nls = DeviceNewton(sp), DeviceNewton(sp)
        x_tr, x_ls = _cuda(x_np), _cuda(x_np)
        same = torch.ones(S, dtype=torch.bool, device="cuda")
        ever = torch.zeros(S, dtype=torch.bool, device="cuda")
        for t in range(12):
            a = ntr.tr_step(x_tr, c1, c2, 2, c3=c3, max_iter=10)
            b = nls.trls_step(x_ls, c1, c2, 2, c3=c3, max_iter=10)
            same &= (a.alpha == 1) | (a.status == N_CONVERGED)
            eq = (_bits(torch, a, S) == _bits(torch, b, S)).all(1)
            assert eq[same].all(), (c3, t)
            moved = torch.zeros(S, device="cuda").index_add_(0, sid, (x_tr != x_ls).any(1).float())
            assert (moved[same] == 0).all(), (c3, t)
            ever |= (b.alpha > 0) & (b.alpha < 1)
        print(f"c3={c3}: spheres on the trust-region trajectory throughout {int(same.sum())} of {S}, "
              f"spheres that backtracked {int(ever.sum())}")
        assert int(same.sum()) > 0 and int(ever.sum()) > 0


@pytest.mark.gpu
def test_trls_determinism_graphs_and_independence(ext):
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
        res = [nw.trls_step(x, c1, c2, 2, c3=C3, anchor=y, weight=w, **o) for _ in range(N)]
        torch.cuda.synchronize()
        return x, _records(torch, res), sum(int(((r.alpha > 0) & (r.alpha < 1)).sum()) for r in res)

    for y, w in ((None, None), (y0, w0)):
        xa, ra, nb = run(x0, y, w)
        assert nb > 0                                          # the runs below do backtrack
        xb, rb, _ = run(x0, y, w)
        assert torch.equal(xa, xb) and torch.equal(ra, rb)
        other = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(other):
            xc, rc, _ = run(x0, y, w)
        assert torch.equal(xa, xc) and torch.equal(ra, rc)
    # 5 proximal steps captured in one graph (after the first call, which allocates), replayed with new anchor data
    yb, wb, xg = y0.clone(), w0.clone(), x0.clone()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        nw.trls_step(x0.clone(), c1, c2, 2, c3=C3, anchor=yb, weight=wb, **o)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        nw.reset()
        rg = _records(torch, [nw.trls_step(xg, c1, c2, 2, c3=C3, anchor=yb, weight=wb, **o) for _ in range(N)])
    xa, ra, _ = run(x0, y0, w0)
    y1 = _cuda(perturb(pk, sigma_rel=0.03, seed=8))
    x1, r1, _ = run(x0, y1, w0)
    assert not torch.equal(x1, xa)
    for yv, xe, re in ((y0, xa, ra), (y1, x1, r1), (y0, xa, ra)):
        yb.copy_(yv)
        xg.copy_(x0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(xg, xe) and torch.equal(rg, re)
    # another start for sphere 4 (a rough one, which backtracks): every other sphere's trajectory bitwise unchanged
    vo = pk.vert_offsets
    keep = torch.ones(len(x0), dtype=torch.bool, device="cuda")
    keep[vo[4]:vo[5]] = False
    others = torch.arange(S, device="cuda") != 4
    xs0 = x0.clone()
    xs0[vo[4]:vo[5]] += 0.01 * torch.randn_like(xs0[vo[4]:vo[5]])
    nw.reset()
    xs = xs0.clone()
    recs = [nw.trls_step(xs, c1, c2, 2, c3=C3, **o) for _ in range(N)]
    nw.reset()
    xr = x0.clone()
    refs = [nw.trls_step(xr, c1, c2, 2, c3=C3, **o) for _ in range(N)]
    assert torch.equal(xs[keep], xr[keep]) and not torch.equal(xs[~keep], xr[~keep])
    for p, q in zip(recs, refs):
        for f in p._fields:
            assert torch.equal(getattr(p, f)[others], getattr(q, f)[others]), f


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(warps_per_cta=8), dict(force_global=True), dict(psd=True)], ids=["w8", "global", "psd"])
def test_trls_handle_variants_and_orphans(ext, kw):
    """Orphan vertices never move; E falls on every sphere; a frozen (CONVERGED) sphere does not move; with proximal
    weights, a NaN (sphere 0) and a negative one (sphere 1) freeze just that sphere as STALLED.  "psd": over a
    projected-Hessian workspace."""
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
    for t in range(4):
        r = nw.trls_step(x, c1, c2, 2)
        assert torch.equal(x[orph], x0[orph]) and (r.delta <= 0).all() and not torch.isnan(x).any()
        assert torch.isin(r.alpha, torch.tensor(ALPHAS + [0.0], device="cuda")).all()
    e1 = sp.energy_grad_spheres(x, c1, c2, 2, want_grad=False)[2]
    assert ((c1 * e1.smooth + c2 * e1.barrier) < (c1 * e0.smooth + c2 * e0.barrier)).all()
    if psd:
        assert not torch.isin(r.pcg_status, torch.tensor([NEGCURV, NEGCURV_FIRST], device="cuda")).any()
    # a frozen sphere: gtol between sphere 2's |g| and the others' converges (and freezes) just that one
    nw.reset()
    x = x0.clone()
    g = nw.trls_step(x.clone(), c1, c2, 2, max_iter=1).grad_norm
    nw.reset()
    lo = int(torch.argmin(g))
    gtol = float(g[lo]) * 1.0001
    assert (g[torch.arange(S, device="cuda") != lo] > gtol).all()
    r = nw.trls_step(x, c1, c2, 2, gtol=gtol)
    assert int(r.status[lo]) == N_CONVERGED and torch.equal(x[sid == lo], x0[sid == lo])
    xf = x.clone()
    r = nw.trls_step(x, c1, c2, 2, gtol=gtol)
    assert torch.equal(x[sid == lo], xf[sid == lo]) and float(r.alpha[lo]) == 0.0 and float(r.grad_norm[lo]) == 0.0
    if psd:
        return
    nw.reset()
    x = x0.clone()
    y = (x0 + 0.01 * torch.randn_like(x0)).contiguous()
    w = torch.tensor([float("nan"), -1e-3, 1e-3], device="cuda")
    for t in range(4):
        r = nw.trls_step(x, c1, c2, 2, anchor=y, weight=w)
        assert torch.equal(x[orph], x0[orph])
        assert r.status[:2].tolist() == [STALLED, STALLED] and r.alpha[:2].tolist() == [0.0, 0.0]
    frozen = (sid < 2) & ~orph
    assert torch.equal(x[frozen], x0[frozen]) and not torch.equal(x[sid == 2], x0[sid == 2])


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_trls_convergence_mixed_pack(ext, amips):
    """The mixed 64 x 4096 pack through SmoothnessBarrierEnergy.newton_step with FLAGS.newton_method = "trls", as
    test_tr_convergence_mixed_pack: every step's change is <= 0 and agrees with a fresh sphere_stats launch; every
    backtracked step has the Armijo decrease delta <= -sigma alpha b.d; the quiet spheres gain no inverted tet and each
    ends CONVERGED within the fp64 reference's step count plus GPU_SLACK; the rough spheres gain at most
    MAX_ROUNDING_FLIPS tets per step and lose inverted tets overall."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("mixed")
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000,
                                                        amips_coeff=C3 if amips else 0.0, deterministic=True, newton_method="trls"))
    x = torch.nn.Parameter(_cuda(x_np))
    it = 0
    e_start, inv_start = _stats(E, x, it)
    g0 = E.newton_step(x.detach().clone(), it, max_iter=1).grad_norm
    E.device_newton.reset()
    quiet = torch.arange(pk.num_spheres, device="cuda") % 4 != 0
    gtol = 1e-3 * float(g0[quiet].min())
    acc = torch.zeros(pk.num_spheres, dtype=torch.float64, device="cuda")
    inv_prev = inv_start
    n = TRLS_REF_STEPS["amips" if amips else "plain"] + GPU_SLACK
    done, n_back = None, 0
    sigma = f32(TRLS_OPTS["sigma"])
    for t in range(n):
        r = E.newton_step(x, it, gtol=gtol)
        assert (r.delta <= 0).all(), t
        back = (r.alpha > 0) & (r.alpha < 1)
        n_back += int(back.sum())
        assert (r.delta.double()[back] <= -sigma * r.alpha.double()[back] * r.b_dot_d.double()[back]).all(), t
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
    print(f"amips={amips}: quiet spheres converged after {done} steps (allowed {n}); backtracked steps {n_back}; "
          f"status {r.status.cpu().tolist()}; radius {float(r.radius.min()):.3e}..{float(r.radius.max()):.3e}")
    assert (r.status[quiet] == N_CONVERGED).all(), r.status
    assert n_back > 0


@pytest.mark.gpu
def test_trls_bookkeeping_and_argument_errors(ext):
    torch = _torch()
    from tssplat_b200 import _capi
    from tssplat_b200.newton import DeviceNewton, DevicePCG
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    ws = DevicePCG(sp)
    nw, ntr = DeviceNewton(sp, ws), DeviceNewton(sp, DevicePCG(sp))
    S = nw.n_spheres
    nw0 = nw.device_bytes
    c1, c2 = COEF
    x = _cuda(x_np)
    E = _capi.TSB_E_INVALID
    st = torch.cuda.current_stream().cuda_stream
    L = _capi.lib
    terms = _capi.tsb_terms_t(c1=c1, c2=c2, order=2, c3=0.0)
    # the first step allocates: refused inside a capture (which survives), then made outside it
    graph = torch.cuda.CUDAGraph()
    g = x.clone()
    with torch.cuda.graph(graph):
        g.add_(1.0)
        with pytest.raises(RuntimeError, match="capture"):
            nw.trls_step(g, c1, c2, 2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(g, x + 1.0) and nw.device_bytes == nw0
    z = x.clone()
    o = nw.tr_options()
    for bad in (dict(n_alpha=1), dict(n_alpha=0), dict(n_alpha=9), dict(sigma=0.0), dict(sigma=0.5), dict(sigma=-1e-4),
                dict(sigma=float("nan")), dict(reserved=1)):
        bt = _capi.tsb_newton_backtrack_t(n_alpha=bad.get("n_alpha", 8), sigma=bad.get("sigma", 1e-4))
        if "reserved" in bad:
            bt.reserved[5] = 1
        assert L.tsb_newton_tr_step_ex(nw._nw, z.data_ptr(), None, None, C.byref(terms), C.byref(o), C.byref(bt), None, st) == E, bad
    bt = _capi.tsb_newton_backtrack_t(n_alpha=8, sigma=1e-4)
    for bad in (dict(max_iter=0), dict(radius_min=0.0), dict(accept=0.25), dict(eta=1.5)):       # the trust-region options' rules
        ob = nw.tr_options(**bad)
        assert L.tsb_newton_tr_step_ex(nw._nw, z.data_ptr(), None, None, C.byref(terms), C.byref(ob), C.byref(bt), None, st) == E, bad
    ob = nw.tr_options()
    ob.reserved[6] = 1
    assert L.tsb_newton_tr_step_ex(nw._nw, z.data_ptr(), None, None, C.byref(terms), C.byref(ob), C.byref(bt), None, st) == E
    y, w = x.clone(), torch.full((S,), 1e-3, device="cuda")
    for args in ((None, z.data_ptr(), None, None, C.byref(terms), C.byref(o)),
                 (nw._nw, None, None, None, C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), y.data_ptr(), None, C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), z.data_ptr(), w.data_ptr(), C.byref(terms), C.byref(o)),
                 (nw._nw, z.data_ptr(), None, None, C.byref(terms), None),
                 (nw._nw, z.data_ptr(), None, None, C.byref(_capi.tsb_terms_t(c1=c1, c2=c2, order=3)), C.byref(o))):
        assert L.tsb_newton_tr_step_ex(*args, C.byref(bt), None, st) == E
    with pytest.raises(TypeError):
        nw.trls_options(tau=1.0)
    with pytest.raises(TypeError):
        nw.tr_options(sigma=1e-4)
    with pytest.raises(ValueError):
        nw.minimize(z, 1, c1, c2, 2, method="cg")
    torch.cuda.synchronize()
    assert torch.equal(z, x) and nw.device_bytes == nw0
    # after the first step: exactly the trust-region step's device memory
    nw.trls_step(z, c1, c2, 2)
    ntr.tr_step(x.clone(), c1, c2, 2)
    assert nw.device_bytes == ntr.device_bytes > nw0
    nw.trls_step(z.clone(), c1, c2, 2, anchor=y, weight=w)
    ntr.tr_step(x.clone(), c1, c2, 2, anchor=y, weight=w)
    assert nw.device_bytes == ntr.device_bytes
    # later calls can be captured: a graph of one step replays the eager step bitwise
    nw.reset()
    xe = x.clone()
    re = _records(torch, [nw.trls_step(xe, c1, c2, 2, n_alpha=4)])
    xg = x.clone()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        nw.reset()
        rg = _records(torch, [nw.trls_step(xg, c1, c2, 2, n_alpha=4)])
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(xg, xe) and torch.equal(rg, re)


@pytest.mark.gpu
def test_module_trls_route(ext):
    """FLAGS.newton_method = "trls" routes newton_step and prox_step to the backtracking trust-region step."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    from tssplat_b200.newton import DeviceNewton, NewtonTRStepResult
    pk, x_np = _pack("small")
    flags = dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000, deterministic=True)
    it = 5
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, dict(flags, newton_method="trls"))
    xa = torch.nn.Parameter(_cuda(x_np))
    ra = E.newton_step(xa, it)
    E2 = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    nw = DeviceNewton(E2.tet_sp)
    c1, c2 = E2.coeff_scheduler(it)
    z = _cuda(x_np)
    rz = nw.trls_step(z, c1, c2, E2.order_at(it))
    assert isinstance(ra, NewtonTRStepResult) and torch.equal(z, xa.detach()) and torch.equal(ra.radius, rz.radius)
    y = _cuda(perturb(pk, sigma_rel=0.01, seed=5))
    r = E.prox_step(xa, y, it, 1e-2, n_steps=3, max_iter=15)
    assert isinstance(r, NewtonTRStepResult) and (r.alpha > 0).any()
    nw.reset()
    n, r2 = nw.minimize(z, 3, c1, c2, E2.order_at(it), anchor=y, weight=1e-2, method="trls", max_iter=15)
    assert n == 3 and torch.equal(z, xa.detach()) and torch.equal(r2.radius, r.radius)
    with pytest.raises(TypeError):
        E.newton_step(xa, it, tau=1.0)
