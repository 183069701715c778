"""The proximal Newton step: tsb_newton_prox_step, DeviceNewton.step/minimize(anchor=, weight=) and
SmoothnessBarrierEnergy.prox_step, which minimise Phi_c(x) = E_c(x) + (w_c / 2) |x_c - y_c|^2 per sphere.

CPU: the damped rule's proximal terms with known answers.  GPU: w = 0 is tsb_newton_step bitwise; convergence and the
anchor bound on the mixed 64 x 4096 pack against the fp64 oracle; argument errors and bookkeeping; the module route.
What the proximal step shares with the other Newton steps (the fp64 reference, whose fixed point is checked against
scipy's trust-region Newton-CG and which pins the step counts; the step against its composition; determinism, graph
replays with new anchors and weights, independence; handle variants, orphans and invalid weights) runs
through the shared checks of _newton_checks."""
import ctypes as C

import numpy as np
import pytest

from _newton_checks import check_composition, check_determinism, check_handle_variants, check_reference
from _newton_model import (ACTIVE, C3, CHUNK, COEF, GPU_SLACK, N_CONVERGED, OPTS, PROX_REF_STEPS, STALLED, Fp64Problem,  # noqa: F401
                           _cuda, _handle, _pack, _records, _torch, _weights, decide_damped, ext, f32, init_shift, new_state)
from tssplat_b200.mesh import perturb


# ---------------------------------------------------------------------------------------------------------------------
# the proximal rule in numpy


_BASE = dict(g=1.0, bd=1.0, dHd=1.5, mu_f=1.0, dd=1.0, dE=[-0.5] + [-0.3 * 2.0 ** -k for k in range(1, 8)], ahat=np.inf)


def _prule(s, w=0.0, dx=0.0, **kw):
    a = dict(_BASE, o=dict(OPTS))
    a.update(kw)
    return decide_damped(s, w=w, dx=dx, **a)


def test_prox_rule_known_answers():
    # w = 0 is the plain rule, on every branch its known answers exercise: d.(x - y) drops out
    cases = [dict(dE=[-0.75] + [-0.1] * 7), dict(dE=[-1.5] + [-0.1] * 7), dict(dE=[0.2, -0.2] + [-0.01] * 6),
             dict(ahat=np.float32(0.3)), dict(dE=[1.0] * 8), dict(bd=-1.0, dE=[-5.0] * 8), dict(bd=1.0, dHd=10.0, dd=0.0),
             dict(g=f32(1e-3), o=dict(OPTS, gtol=1e-3))]
    for kw in cases:
        s1, s2 = dict(mu=3.0, nu=2.0, status=ACTIVE), dict(mu=3.0, nu=2.0, status=ACTIVE)
        a = dict(_BASE, o=dict(OPTS))
        a.update(kw)
        assert _prule(s1, w=0.0, dx=0.7, **kw) == decide_damped(s2, **a) and s1 == s2, kw
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
    sh = init_shift(st, [np.float32(4.0), np.float32(1.0)], OPTS, [np.float32(0.5), np.float32(np.nan)])
    assert st[0]["mu"] == f32(1e-3) * 4.5 and sh[0] == np.float32(st[0]["mu"] + 0.5)
    assert st[1]["mu"] == f32(1e-3) * 1.0 and sh[1] == np.float32(st[1]["mu"])
    # an unusable weight: no step, STALLED, mu untouched, and it stays frozen
    for w in (float("nan"), float("inf"), -1e-3):
        s = dict(mu=1.0, nu=2.0, status=ACTIVE)
        assert _prule(s, w=w, dE=[-0.75] + [-0.1] * 7) == (0.0, -1, 0.0, 0.0)
        assert s == dict(mu=1.0, nu=2.0, status=STALLED)
        assert _prule(s, w=1.0, dE=[-0.75] + [-0.1] * 7) == (0.0, -1, 0.0, 0.0) and s["status"] == STALLED


# ---------------------------------------------------------------------------------------------------------------------
# GPU


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


# ---------------------------------------------------------------------------------------------------------------------
# the checks every Newton step shares (_newton_checks)


@pytest.mark.parametrize("scale", ["small", "large"])
def test_prox_reference_mixed_pack(scale):
    check_reference("prox", scale)


@pytest.mark.gpu
@pytest.mark.parametrize("c3", [0.0, C3], ids=["amips-off", "amips-on"])
def test_prox_step_equals_its_composition(ext, c3):
    check_composition(ext, "prox", c3, prox=True)


@pytest.mark.gpu
def test_prox_determinism_graphs_and_independence(ext):
    check_determinism(ext, "prox")


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["w8", "w16", "global"])
def test_prox_handle_variants_orphans_and_invalid_weights(ext, variant):
    check_handle_variants(ext, "prox", variant)
