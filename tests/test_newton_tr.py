"""The trust-region Newton step: tsb_pcg_solve_tr (Steihaug-Toint CG inside a per-sphere radius in the preconditioner
norm), tsb_newton_tr_step, DevicePCG.solve(radius=), DeviceNewton.tr_step / minimize(method="tr") and
SmoothnessBarrierEnergy with FLAGS.newton_method = "tr".

CPU: _newton_model's batched fp64 Steihaug-Toint state machine against dense per-sphere problems (SPD and indefinite):
its M-norm recurrences against the directly computed |d_k|_M, monotone growth, the boundary step, the Cauchy decrease,
and the infinite radius as the plain PCG reference; the trust-region rule with known answers.  GPU: radius +inf is
tsb_pcg_solve_ex bitwise; finite radii are respected in the M-norm and negative curvature is followed to the boundary;
bookkeeping and argument errors; the module route.  What the trust-region step shares with the other Newton steps (the
fp64 reference, plain and proximal, which pins the step counts; the step against its composition; determinism, graph
replays and independence; handle variants, orphans and the projected Hessian; convergence on the mixed 64 x 4096 pack)
runs through the shared checks of _newton_checks."""
import ctypes as C

import numpy as np
import pytest

from _newton_checks import (check_composition, check_convergence, check_determinism, check_handle_variants,
                            check_reference)
from _newton_model import (ACTIVE, BOUNDARY, C3, CHUNK, COEF, CONVERGED, N_CONVERGED, NEGCURV, NEGCURV_BOUNDARY,  # noqa: F401
                           NEGCURV_FIRST, STALLED, TR_OPTS, _cuda, _handle, _labels, _m_norm, _pack, _seg_sum,
                           _shuffled_mesh, _spd, _sphere_max_diag, _torch, batched_pcg_reference, batched_steihaug,
                           decide_tr, ext, f32, init_radius, new_state)
from tssplat_b200.mesh import perturb


# ---------------------------------------------------------------------------------------------------------------------
# the solve and the rule in numpy


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
    return decide_tr(s, **dict(a, dphi=[a["dphi"]]))


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
    st = new_state(3)
    r = init_radius(st, [4.0, 0.0, 1e30], dict(TR_OPTS, radius_init=0.5, radius_min=1e-3, radius_max=1e6))
    assert r.tolist() == [1.0, f32(1e-3), f32(1e6)]


# ---------------------------------------------------------------------------------------------------------------------
# GPU


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


# ---------------------------------------------------------------------------------------------------------------------
# the checks every Newton step shares (_newton_checks)


@pytest.mark.parametrize("kind", ["plain", "amips", "small", "large"])
def test_tr_reference_mixed_pack(kind):
    check_reference("tr", kind)


@pytest.mark.gpu
@pytest.mark.parametrize("prox", [False, True], ids=["plain", "prox"])
def test_tr_step_equals_its_composition(ext, prox):
    check_composition(ext, "tr", C3, prox)


@pytest.mark.gpu
def test_tr_determinism_graphs_and_independence(ext):
    check_determinism(ext, "tr")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["w8", "w16", "global", "psd"])
def test_tr_handle_variants_and_orphans(ext, variant):
    check_handle_variants(ext, "tr", variant)


@pytest.mark.gpu
@pytest.mark.parametrize("amips", [False, True], ids=["amips-off", "amips-on"])
def test_tr_convergence_mixed_pack(ext, amips):
    check_convergence(ext, "tr", amips)
