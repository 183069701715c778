"""The checks every device Newton step shares, written once and run per method by each method's test module: the damped
step (lm: DeviceNewton.step), the proximal step (prox: step with an anchor and weights), projected Newton (psd: the
damped step over a projected-Hessian workspace), the trust-region step (tr: tr_step) and the backtracking trust-region
step (trls: trls_step).  Not a test module.

CPU: the fp64 reference of each method (_newton_model.reference) on the small mixed pack: the objective never
increases and its change is the record's, the step counts each method is pinned to, stationarity at the fixed point
and, with an anchor, the fixed point against scipy's trust-region Newton-CG.  GPU: one step against the public calls
composed with the numpy rule; determinism, another stream, CUDA graph replays (with new anchors and weights) and
per-sphere independence; handle variants, orphans and unusable weights; convergence on the mixed 64 x 4096 pack within
the fp64 reference's step count plus GPU_SLACK."""
import numpy as np

from _newton_model import (ALPHAS, BOUNDARY, C3, COEF, GPU_SLACK, MAX_ROUNDING_FLIPS, N_CONVERGED, NEGCURV,
                           NEGCURV_BOUNDARY, NEGCURV_FIRST, OPTS, REF_STEPS, STALLED, STEPS, TR_OPTS, TR_REF_STEPS,
                           TRLS_OPTS, TRLS_REF_STEPS, _cuda, _handle, _labels, _p_apply, _pack, _records, _seg_sum,
                           _shuffled_mesh, _torch, _weights, compose, converged_at, f32, new_state, reference_run)
from tssplat_b200.mesh import perturb


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references (CPU)


def check_reference(method, variant):
    """One fp64 reference run of REFERENCE_RUNS."""
    from scipy.optimize import minimize
    from test_hvp import hvp
    P, x0, w, o, must, pinned, x, hist = reference_run(method, variant)
    y = x0.reshape(-1)
    wv = np.repeat(w, np.diff(P.vo) * 3) if w is not None else 0.0
    assert hist[0][0]["inv0"] > 0 and all(h["inv0"] == 0 for h in hist[0][1:])     # sphere 0 starts with inverted tets
    if method == "lm":                                                             # no tet with J > 0 inverts
        from oracle.tet_energy_oracle import _det3
        J0 = _det3((P.orc.G @ y).reshape(-1, 3, 3))
        J = _det3((P.orc.G @ x).reshape(-1, 3, 3))
        assert not ((J0 > 0) & (J <= 0)).any()
    n_back = 0
    after_all = P.objective(x, y, w)
    for t, step in enumerate(hist):              # the objective never increases; its change is the record's
        nxt = hist[t + 1] if t + 1 < len(hist) else None
        for s, r in enumerate(step):
            after = nxt[s]["phi0"] if nxt else after_all[s]
            assert after <= r["phi0"] + 1e-12 * abs(r["phi0"]), (t, s)
            assert abs((after - r["phi0"]) - r["delta"]) <= 1e-9 * abs(r["phi0"]), (t, s)
            if 0.0 < r["alpha"] < 1.0:           # a shorter step: Armijo below the inversion bound
                n_back += 1
                assert r["alpha"] < f32(o["eta"]) * r["ahat"] and r["delta"] <= -f32(o["sigma"]) * r["alpha"] * r["bd"], (t, s)
            if nxt and (method in ("lm", "tr") or (method == "trls" and s > 0)):
                assert nxt[s]["inv0"] <= r["inv0"]
            if method == "psd":                  # the projected solve never stops at negative curvature
                assert r["pcg"] not in (NEGCURV, NEGCURV_FIRST), (t, s, r["pcg"])
    conv = converged_at(hist, P.S)
    print(f"{method} {variant}: converged at steps {conv}, backtracked steps {n_back}, "
          f"alpha {[[h['alpha'] for h in step] for step in hist]}, solve statuses {sorted({h['pcg'] for st in hist for h in st})}")
    assert all(conv[s] is not None and conv[s] <= pinned for s in must), conv
    if method in ("tr", "trls"):
        assert {h["pcg"] for step in hist for h in step} & {BOUNDARY, NEGCURV_BOUNDARY}        # the radius was active somewhere
    if method == "trls":
        assert n_back > 0
        assert all(conv[s] <= TR_REF_STEPS[variant] for s in range(1, P.S)), conv     # quiet spheres: within the TR counts
        if variant == "plain":
            assert hist[-1][0]["inv0"] == 0
    if method == "psd":                          # the spheres that need not converge keep descending
        for s in set(range(P.S)) - set(must):
            assert all(step[s]["delta"] < 0 for step in hist), s

    def jac(z):
        return P.grad(z) + wv * (z - y)

    gx = jac(x)
    for s in must:                                                          # stationary to gtol
        assert np.linalg.norm(gx[3 * P.vo[s]:3 * P.vo[s + 1]]) <= o["gtol"] * (1 + 1e-6), s
    if w is None:
        return
    # the fixed point against an independent minimiser of Phi: scipy's trust-region Newton-CG with the oracle's fp64
    # gradient and the matrix-form HVP, from the same start.  Both points are stationary to gtol, and Phi_c is
    # w_c-strongly convex where H_c is PSD, so per sphere |x_c - x*_c| <= (|grad Phi_c(x)| + |grad Phi_c(x*)|) / w_c, and
    # Phi_c agrees to that distance times the gradients
    ref = minimize(lambda z: float(P.objective(z, y, w).sum()), y.copy(), jac=jac,
                   hessp=lambda z, p: hvp(P.orc, z, p, P.c1, P.c2, P.order).reshape(-1) + wv * p, method="trust-ncg",
                   options=dict(gtol=1e-3 * o["gtol"], maxiter=500))
    others = [ref.x]
    if method == "psd":                          # and the exact mode's fixed point
        others.append(reference_run("prox", variant)[6])
    for other in others:
        go = jac(other)
        for s in must:
            sl = slice(3 * P.vo[s], 3 * P.vo[s + 1])
            gs, grs = np.linalg.norm(gx[sl]), np.linalg.norm(go[sl])
            dist = np.linalg.norm(x[sl] - other[sl])
            print(f"sphere {s}: |x - x*| = {dist:.3e}, bound {(gs + grs) / w[s]:.3e}")
            assert dist <= (gs + grs) / w[s], (s, dist, (gs + grs) / w[s])
            if method == "prox":
                phis, phir = P.objective(x, y, w)[s], P.objective(other, y, w)[s]
                assert abs(phis - phir) <= (gs + grs) * (gs + grs) / w[s] + 1e-12 * abs(phir), (s, phis, phir)
    if method == "prox" and variant == "large":  # the dominant weight holds x near the anchor; the small one does not
        xs = reference_run("prox", "small")[6]
        assert np.abs(x - y).max() < 0.2 * np.abs(xs - y).max()


# ---------------------------------------------------------------------------------------------------------------------
# GPU


def _step(nw, method, x, c1, c2, c3=0.0, y=None, w=None, **o):
    """One step of method on DeviceNewton nw (an anchor for prox, optional for tr and trls)."""
    run = {"tr": nw.tr_step, "trls": nw.trls_step}.get(method, nw.step)
    return run(x, c1, c2, 2, c3=c3, anchor=y, weight=w, **o)


def check_composition(ext, method, c3, prox):
    """Six (damped) or eight (trust-region) steps on the small pack against the public calls composed with the numpy rule
    (on the method's workspace: a projected one multiplies by H+): bitwise the same x, the same alpha and status, mu to
    fp64 rounding or the radius to 1e-5; every shorter trust-region step satisfies the Armijo decrease below eta alpha^."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    step = STEPS[method]
    damped = step.kind == "damped"
    pk, x_np = _pack("small")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    sid_np, orph_np, S = _labels(pk.verts, pk.tets)
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    nw = DeviceNewton(sp, hessian="psd" if step.projected else None)
    c1, c2 = COEF
    o = dict(OPTS if damped else TRLS_OPTS if step.backtrack else TR_OPTS, gtol=0.05)
    x1 = _cuda(x_np)
    y = w = None
    if prox:
        # the backtracking step is anchored at the start: the pull holds the rough sphere near its inverted tets, so it
        # backtracks; the others a little off it
        y = x1.clone() if method == "trls" else _cuda(perturb(pk, sigma_rel=0.01, seed=5))
        w = _weights(torch, sp.hess_diag(x1, c1, c2, 2, c3=c3), sid, orph, S, [1e-3, 1e-1, 1.0])
    if not damped:
        # the initial radius clamped to radius_max on every sphere, so that it does not depend on how b^T P b is summed
        # (the kernel forms P b in fp32); well below every sphere's radius_init |b|_P, so the radius binds at the start
        _, g = sp.energy_grad(x1, c1, c2, 2, c3=c3)
        inv = nw.pcg.set_blocks(sp.hess_diag(x1, c1, c2, 2, c3=c3), want_inverse=True)
        gd = g.double()
        o["radius_max"] = 0.1 * float(_seg_sum(torch, (gd * _p_apply(inv, gd)).sum(1)[~orph], sid[~orph], S).sqrt().min())
    x2 = x1.clone()
    st = new_state(S)
    seen, full, back, prev = set(), 0, 0, None
    for t in range(6 if damped else 8):
        r = _step(nw, method, x1, c1, c2, c3, y, w, **o)
        x2, out = compose(torch, sp, nw.pcg, x2, st, c1, c2, c3, o, step, sid, orph, S, y=y, w=w, radius_after=prev)
        assert torch.equal(x1, x2), t
        alpha = r.alpha.cpu().tolist()
        assert alpha == [q["alpha"] for q in out], t
        assert r.status.cpu().tolist() == [s["status"] for s in st], t
        if damped:
            assert r.k.cpu().tolist() == [q["k"] for q in out], t
            assert np.allclose(r.mu.cpu().numpy(), [s["mu"] for s in st], rtol=1e-12, atol=0), t
            if method == "prox":
                took = np.array([q["k"] >= 0 for q in out])
                assert np.allclose(r.delta.cpu().numpy()[took], [q["delta"] for q in out if q["k"] >= 0], rtol=1e-5, atol=0), t
        else:
            assert np.allclose(r.radius.cpu().numpy(), [s["radius"] for s in st], rtol=1e-5, atol=0), t
            assert np.allclose(r.pred.cpu().numpy(), [q["pred"] for q in out], rtol=1e-6, atol=0), t
            if method == "tr":
                assert np.allclose(r.d_norm.cpu().numpy() ** 2, [q["dMd"] for q in out], rtol=1e-4, atol=0), t
            delta = r.delta.cpu().numpy()
            for c, q in enumerate(out):
                if 0.0 < q["alpha"] < 1.0:
                    k = ALPHAS.index(q["alpha"])
                    assert q["alpha"] < f32(o["eta"]) * q["ahat"] and q["dphi"][k] <= -f32(o["sigma"]) * q["alpha"] * q["bd"], (t, c)
                    assert abs(delta[c] - q["dphi"][k]) <= 1e-6 * abs(q["dphi"][k]) + 1e-12, (t, c)
            prev = r.radius.cpu().numpy()
            full += alpha.count(1.0)
            back += sum(0.0 < a < 1.0 for a in alpha)
        seen |= set(r.status.cpu().tolist())
    print(f"{method} c3={c3} prox={prox}: states seen {sorted(seen)}, full steps {full}, backtracked {back}")
    assert N_CONVERGED in seen
    if method == "lm":
        assert int((r.status == N_CONVERGED).sum()) >= 1         # converged spheres at the last step
    if not damped:
        assert full > 0
    if method == "trls":
        assert back > 0


# lm steps without an anchor, prox with one; tr and trls both
_ANCHORED = {"lm": (False,), "prox": (True,), "tr": (False, True), "trls": (False, True)}


def check_determinism(ext, method):
    """On the mixed 64 x 4096 pack: ten steps twice and on another stream give bitwise the same x and records; ten
    steps captured in one CUDA graph (with anchor and weight buffers where the method takes them) replay bitwise, also
    after new anchor and weight data is copied into the buffers; another start, anchor or weight for sphere 4 (a rough
    sphere, which the backtracking step backtracks) leaves every other sphere's trajectory bitwise unchanged."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    pk, x_np = _pack("mixed")
    sp = _handle(ext, pk.verts, pk.tets, enable_amips=True, deterministic=True)
    S = pk.num_spheres
    sid = torch.from_numpy(np.repeat(np.arange(S), np.diff(pk.vert_offsets))).cuda()
    nw = DeviceNewton(sp)
    c1, c2 = COEF
    o = dict(max_iter=10)
    N = 10
    x0 = _cuda(x_np)
    y0 = _cuda(perturb(pk, sigma_rel=0.02, seed=7))
    w0 = _weights(torch, sp.hess_diag(x0, c1, c2, 2, c3=C3), sid, torch.zeros_like(sid, dtype=torch.bool), S, [1e-3, 1e-2, 1e-1])

    def steps(x, y, w):
        return [_step(nw, method, x, c1, c2, C3, y, w, **o) for _ in range(N)]

    def run(x_start, y=None, w=None):
        nw.reset()
        x = x_start.clone()
        res = steps(x, y, w)
        torch.cuda.synchronize()
        return x, _records(torch, res), sum(int(((r.alpha > 0) & (r.alpha < 1)).sum()) for r in res)

    for anchored in _ANCHORED[method]:
        y, w = (y0, w0) if anchored else (None, None)
        xa, ra, nb = run(x0, y, w)
        if method == "trls":
            assert nb > 0                                          # the runs below do backtrack
        xb, rb, _ = run(x0, y.clone() if anchored else None, w.clone() if anchored else None)
        assert torch.equal(xa, xb) and torch.equal(ra, rb)
        other = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(other):
            xc, rc, _ = run(x0, y, w)
        assert torch.equal(xa, xc) and torch.equal(ra, rc)
    # N steps captured in one graph (after a first call, which allocates), with anchor and weight buffers where the
    # method takes an anchor, replayed after new data is copied into them
    anchored = True in _ANCHORED[method]
    yb, wb = (y0.clone(), w0.clone()) if anchored else (None, None)
    xg = x0.clone()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        _step(nw, method, x0.clone(), c1, c2, C3, yb, wb, **o)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        nw.reset()
        rg = _records(torch, steps(xg, yb, wb))
    replays = [(y0, w0, xa, ra)] * 2
    if anchored:
        y1 = _cuda(perturb(pk, sigma_rel=0.03, seed=8))
        w1 = (w0 * torch.linspace(0.5, 2.0, S, device="cuda")).contiguous()
        x1, r1, _ = run(x0, y1, w1)
        assert not torch.equal(x1, xa)
        replays = [(y0, w0, xa, ra), (y1, w1, x1, r1), (y0, w0, xa, ra)]
    for yv, wv, xe, re in replays:
        if anchored:
            yb.copy_(yv)
            wb.copy_(wv)
        xg.copy_(x0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(xg, xe) and torch.equal(rg, re)
    # another start (without an anchor), anchor or weight for sphere 4 only: every other sphere's trajectory bitwise
    # unchanged
    vo, k = pk.vert_offsets, 4
    keep = torch.ones(len(x0), dtype=torch.bool, device="cuda")
    keep[vo[k]:vo[k + 1]] = False
    others = torch.arange(S, device="cuda") != k
    xs0, y2, w2 = x0.clone(), y0.clone(), w0.clone()
    xs0[vo[k]:vo[k + 1]] += 0.01 * torch.randn_like(xs0[vo[k]:vo[k + 1]])
    y2[vo[k]:vo[k + 1]] += 0.01 * torch.randn_like(y2[vo[k]:vo[k + 1]])
    w2[k] *= 3.0
    cases = []
    if False in _ANCHORED[method]:
        cases.append((xs0, None, None, None, None))
    if True in _ANCHORED[method]:
        cases += [(x0, y2, w0, y0, w0), (x0, y0, w2, y0, w0)]
    for xv, yv, wv, yr, wr in cases:
        nw.reset()
        xs = xv.clone()
        recs = steps(xs, yv, wv)
        nw.reset()
        xr = x0.clone()
        refs = steps(xr, yr, wr)
        assert torch.equal(xs[keep], xr[keep]) and not torch.equal(xs[~keep], xr[~keep])
        for p, q in zip(recs, refs):
            for f in p._fields:
                assert torch.equal(getattr(p, f)[others], getattr(q, f)[others]), f


_VARIANTS = {"w8": dict(warps_per_cta=8), "w16": dict(warps_per_cta=16), "global": dict(force_global=True), "psd": dict()}


def check_handle_variants(ext, method, variant):
    """The shuffled mesh (500 orphans): orphan vertices never move; without an anchor E falls on every sphere (and a
    frozen CONVERGED sphere does not move under the backtracking step); with proximal weights, a NaN (sphere 0) and a
    negative one (sphere 1) freeze just that sphere as STALLED, unmoved, while the third steps.  "psd": over a
    projected-Hessian workspace."""
    torch = _torch()
    from tssplat_b200.newton import DeviceNewton
    V, T, x_np = _shuffled_mesh()
    kw = _VARIANTS[variant]
    psd = variant == "psd"
    sp = _handle(ext, V, T, deterministic=True, **kw)
    assert sp.info["mode_global"] == int(bool(kw.get("force_global")))
    sid_np, orph_np, S = _labels(V, T)
    assert S == 3
    sid, orph = torch.from_numpy(sid_np).cuda(), torch.from_numpy(orph_np).cuda()
    c1, c2 = COEF
    nw = DeviceNewton(sp, hessian="psd" if psd else None)
    x0 = _cuda(x_np)
    if method != "prox":
        x = x0.clone()
        e0 = sp.energy_grad_spheres(x0, c1, c2, 2, want_grad=False)[2]
        for t in range({"lm": 8, "tr": 1 if psd else 4, "trls": 4}[method]):
            r = _step(nw, method, x, c1, c2)
            assert torch.equal(x[orph], x0[orph]) and (r.delta <= 0).all() and not torch.isnan(x).any()
            if method == "trls":
                assert torch.isin(r.alpha, torch.tensor(ALPHAS + [0.0], device="cuda")).all()
        if method == "tr":
            assert (r.alpha == 1).all() or t > 0
        e1 = sp.energy_grad_spheres(x, c1, c2, 2, want_grad=False)[2]
        assert ((c1 * e1.smooth + c2 * e1.barrier) < (c1 * e0.smooth + c2 * e0.barrier)).all()
        if psd:
            assert not torch.isin(r.pcg_status, torch.tensor([NEGCURV, NEGCURV_FIRST], device="cuda")).any()
    if method == "trls":
        # a frozen sphere: gtol between sphere lo's |g| and the others' converges (and freezes) just that one
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
    if method == "lm" or psd:
        return
    nw.reset()
    x = x0.clone()
    y = (x0 + 0.01 * torch.randn_like(x0)).contiguous()
    w = torch.tensor([float("nan"), -1e-3, 1e-3], device="cuda")
    for t in range(6 if method == "prox" else 4):
        r = _step(nw, method, x, c1, c2, y=y, w=w)
        assert torch.equal(x[orph], x0[orph])
        assert r.status[:2].tolist() == [STALLED, STALLED] and r.alpha[:2].tolist() == [0.0, 0.0]
        if method == "prox":
            assert (r.delta <= 0).all() and not torch.isnan(x).any()
            assert float(r.alpha[2]) > 0 or t > 0
    frozen = (sid < 2) & ~orph
    assert torch.equal(x[frozen], x0[frozen]) and not torch.equal(x[sid == 2], x0[sid == 2])


def _stats(E, x, it):
    st = E.sphere_stats(x, it)
    c1, c2 = E.coeff_scheduler(it)
    return (c1 * st.smooth + c2 * st.barrier + E.amips_coeff * st.amips), st.n_inverted


def check_convergence(ext, method, amips):
    """The mixed 64 x 4096 pack through SmoothnessBarrierEnergy.newton_step with FLAGS.newton_method = method: every
    step's per-sphere energy change is <= 0 and a fresh sphere_stats launch agrees with the start plus the summed deltas
    (with AMIPS on, on the quiet spheres: a rough sphere un-inverts tets to J just above 0, where psi ~ J^(-2/3) makes an
    fp32 re-evaluation of the energy meaningless); every backtracked trust-region step has the Armijo decrease
    delta <= -sigma alpha b.d; the inverted-tet count never grows on the quiet spheres; every quiet sphere ends
    CONVERGED within the fp64 reference's step count plus GPU_SLACK.  On the rough spheres the inversion bound holds for
    the line search's own cubic: a tet whose J sits a few roundings above 0 can still come out inverted once
    x + alpha d is rounded to fp32 (a handful of tets out of ~12 000 over the run, while the rough spheres' inverted
    count falls by hundreds), so there the total must fall and no step may add more than MAX_ROUNDING_FLIPS."""
    torch = _torch()
    from tssplat_b200.energies import SmoothnessBarrierEnergy
    pk, x_np = _pack("mixed")
    flags = dict(smooth_eng_coeff=COEF[0], barrier_coeff=COEF[1], increase_order_iter=1000, amips_coeff=C3 if amips else 0.0,
                 deterministic=True)
    if method != "lm":
        flags["newton_method"] = method
    E = SmoothnessBarrierEnergy(pk.verts, pk.tets, flags)
    x = torch.nn.Parameter(_cuda(x_np))
    it = 0
    e_start, inv_start = _stats(E, x, it)
    g0 = E.newton_step(x.detach().clone(), it, max_iter=1).grad_norm        # |g_c| at the start (x untouched)
    E.device_newton.reset()
    quiet = torch.arange(pk.num_spheres, device="cuda") % 4 != 0
    gtol = 1e-3 * float(g0[quiet].min())
    acc = torch.zeros(pk.num_spheres, dtype=torch.float64, device="cuda")
    inv_prev = inv_start
    n = (REF_STEPS[amips] if method == "lm" else {"tr": TR_REF_STEPS, "trls": TRLS_REF_STEPS}[method]["amips" if amips else "plain"]) \
        + GPU_SLACK
    done, n_back = None, 0
    sigma = f32(TRLS_OPTS["sigma"])
    for t in range(n):
        r = E.newton_step(x, it, gtol=gtol)
        assert (r.delta <= 0).all(), t
        if method == "trls":
            back = (r.alpha > 0) & (r.alpha < 1)
            n_back += int(back.sum())
            assert (r.delta.double()[back] <= -sigma * r.alpha.double()[back] * r.b_dot_d.double()[back]).all(), t
        acc += r.delta.double()
        e, inv = _stats(E, x, it)
        # the line search's deltas are cancellation-free fp32 sums; sphere_stats sums fp32 per-tet energies
        tol = 1e-4 * e_start.abs()
        err = (e - e_start - acc).abs()
        checked = quiet if amips else torch.ones_like(quiet)
        assert (err[checked] <= tol[checked]).all(), (t, float((err / tol)[checked].max()))
        assert (inv[quiet] <= inv_prev[quiet]).all(), t
        up = (inv - inv_prev).clamp(min=0)
        assert int(up.max()) <= MAX_ROUNDING_FLIPS, (t, up)
        if up.any():
            print(f"step {t}: {int(up.sum())} tet(s) newly inverted by fp32 rounding on the rough spheres")
        inv_prev = inv
        if done is None and bool((r.status[quiet] == N_CONVERGED).all()):
            done = t + 1
    assert int(inv[~quiet].sum()) < int(inv_start[~quiet].sum())
    print(f"{method} amips={amips}: quiet spheres converged after {done} steps (allowed {n}); backtracked steps {n_back}; "
          f"status {r.status.cpu().tolist()}; inverted {inv_start[~quiet].sum().item()} -> {inv[~quiet].sum().item()}")
    assert (r.status[quiet] == N_CONVERGED).all(), r.status
    if method == "trls":
        assert n_back > 0
